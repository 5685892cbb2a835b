"""bnn_oracle.py -- NumPy restatement of the fully Bayesian MLP (gpax/models/bnn.py over gpax/models/spm.py).  TEST
INFRASTRUCTURE ONLY (see oracle/__init__.py).

  loglik     sum_{i,o} log N(y_io; z_io, sigma) with z = MLP(X) (tanh hidden layers, linear last layer, bnn.py:55-65),
             d/dsigma, and d/d(W_l, b_l) in the flat layout by dkl_oracle's backward pass from dz = (y - z) / sigma^2
  predict    loc = MLP(X) per weight set and y = loc + sigma * mean_k eps[k] (spm.py:150-154)

Flat layout: per layer W_l [in, out] row-major, then b_l (dkl_oracle.flatten / unflatten)."""
import math

import numpy as np

from . import dkl_oracle as dko


def loglik(X, y, D, widths, flat, sigma, act="tanh"):
    """(value, d value / d sigma, d value / d flat, scale): scale bounds the size of the terms summed into each gradient
    entry (for tolerances relative to it)"""
    X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64)
    layers = dko.unflatten(np.asarray(flat, dtype=np.float64), D, widths)
    H = dko.mlp_forward(X, layers, act)
    r = y - H[-1]
    n = r.size
    value = -0.5 * float(np.sum(r * r)) / sigma ** 2 - n * (math.log(sigma) + 0.5 * math.log(2 * math.pi))
    gsig = float(np.sum(r * r)) / sigma ** 3 - n / sigma
    gflat = dko.backward(H, layers, act, r / sigma ** 2)
    absl = [(np.abs(W), np.abs(b)) for W, b in layers]
    Habs = [np.abs(h) for h in H]
    scale = dko.backward(Habs, absl, act, np.abs(r) / sigma ** 2)      # |1 - h^2| <= 1, so this bounds every term
    return value, gsig, gflat, scale


def predict(X, D, widths, flats, sigma=None, eps=None, act="tanh"):
    """loc [S, P, O] and, given eps [S, n, P, O], y_sampled [S, P, O]"""
    flats = np.atleast_2d(np.asarray(flats, dtype=np.float64))
    loc = np.stack([dko.mlp_forward(X, dko.unflatten(f, D, widths), act)[-1] for f in flats])
    if eps is None:
        return loc, None
    sigma = np.asarray(sigma, dtype=np.float64).reshape(-1, 1, 1)
    return loc, loc + sigma * np.asarray(eps, dtype=np.float64).mean(1)
