"""grad_oracle.py -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

NumPy restatement of the derivatives that jax.grad takes in the reference's optimize_acq (gpax/acquisition/optimize.py:
70-88): the exact-GP posterior mean and variance at a test point differentiated w.r.t. that point, and an acquisition
function of them.  No golden vector can pin a JAX derivative here (JAX does not run), so tests pin these derivatives by
central differences of the oracle's own posterior (`gp_oracle.exact_posterior_chol`, itself pinned to the golden
vectors) and of `acq_oracle`'s acquisitions.

  kernel_dx            d k(x_p, x_i) / d x_p[k] of gpax/kernels/kernels.py:28-117 as written: the clipped
                       X2 - 2 XZ + Z2 distance, Matern's sqrt(r2 + 1e-12) next to its un-eps'd 5/3 r2 term
  posterior_grad       mean, var and their gradients, through the Cholesky factor
  acq_value_grad       EI / UCB / POI / UE at one point from (mean, var) and their gradients; with eps the reference's
                       sample moments (acquisition.py:31-34) of y = mean + sqrt(var) eps, differentiated through
"""
import math

import numpy as np
import scipy.linalg as sla
from scipy.special import ndtr

from . import acq_oracle as ao
from . import gp_oracle as go


def kernel_dx(X_new, X_train, params, kernel="RBF"):
    """D[p, k, i] = d k(X_new[p], X_train[i]) / d X_new[p, k]"""
    Xn, X = go._as2d(X_new), go._as2d(X_train)
    d = Xn.shape[1]
    ell = np.broadcast_to(np.asarray(params["k_length"], dtype=np.float64).reshape(-1), (d,))
    scale = params["k_scale"]
    if kernel == "Periodic":
        a = math.pi * (Xn[:, None, :] - X[None, :, :]) / params["period"]             # [P, N, d]
        k = scale * np.exp(-2 * ((np.sin(a) / ell) ** 2).sum(-1))                       # kernels.py:111-114
        dk = -k[:, :, None] * 2 * math.pi * np.sin(2 * a) / (params["period"] * ell ** 2)
        return dk.transpose(0, 2, 1)
    r2 = go.square_scaled_distance(Xn, X, ell)
    Xs, Zs = Xn / ell, X / ell                                                          # kernels.py:35-40, unclipped
    raw = (Xs ** 2).sum(1)[:, None] - 2 * Xs @ Zs.T + (Zs ** 2).sum(1)[None, :]
    if kernel == "RBF":
        dk_dr2 = -0.5 * scale * np.exp(-0.5 * r2)
    else:
        r = np.sqrt(r2 + 1e-12)
        dk_dr2 = -(5 / 6) * scale * np.exp(-(5 ** 0.5) * r) * (1 + 5 ** 0.5 * r2 / r)
    dk_dr2 = np.where(raw < 0, 0.0, dk_dr2)                                             # clip(0) passes no gradient
    diff = (Xn[:, None, :] - X[None, :, :]) / ell ** 2                                  # [P, N, d]
    return (2 * dk_dr2[:, :, None] * diff).transpose(0, 2, 1)


def posterior_grad(X_train, y_train, X_new, params, kernel="RBF", noiseless=False, jitter=1e-6):
    """(mean [P], var [P], dmean [P, d], dvar [P, d]) of gp.py:253-277's posterior at each test point, w.r.t. that point"""
    kern = go.get_kernel(kernel)
    X, Xn = go._as2d(X_train), go._as2d(X_new)
    mean, var = go.exact_posterior_chol(X, y_train, Xn, params, kernel, noiseless, diag_only=True, jitter=jitter)
    K = kern(X, X, params, params["noise"], jitter=jitter)
    L = sla.cholesky(K, lower=True)
    k_pX = kern(Xn, X, params, jitter=0.0)
    V = sla.solve_triangular(L, k_pX.T, lower=True)                                      # [N, P]
    w = sla.solve_triangular(L, np.asarray(y_train, dtype=np.float64), lower=True)
    D = kernel_dx(Xn, X, params, kernel)                                                 # [P, d, N]
    P, d, N = D.shape
    LD = sla.solve_triangular(L, D.reshape(P * d, N).T, lower=True).T.reshape(P, d, N)
    dmean = LD @ w
    dvar = -2 * np.einsum("pkn,np->pk", LD, V)
    return mean, var, dmean, dvar


def _moments_grad(mean, var, dmean, dvar, eps):
    """(M, V, dM, dV): the moments themselves (eps None, one draw) or the sample moments of y = mean + sqrt(var) eps"""
    mean, var = np.atleast_1d(mean).astype(float), np.atleast_1d(var).astype(float)
    dmean, dvar = np.atleast_2d(dmean), np.atleast_2d(dvar)
    if eps is None:
        return mean[0], var[0], dmean[0], dvar[0]
    eps = np.asarray(eps, dtype=np.float64).reshape(mean.size, -1)
    S, n = eps.shape
    ys, dys = [], []
    for s in range(S):
        sd = np.sqrt(var[s])
        for i in range(n):
            ys.append(mean[s] + sd * eps[s, i])
            dys.append(dmean[s] + eps[s, i] * dvar[s] / (2 * sd))
    y, dy = np.array(ys), np.array(dys)
    M, V = ao.moments_from_samples(y[:, None])
    M, V = M[0], V[0]
    dM = dy.mean(0)
    dV = (2 / y.size) * ((y - M)[:, None] * (dy - dM)).sum(0)
    return M, V, dM, dV


def acq_value_grad(kind, mean, var, dmean, dvar, eps=None, best_f=None, param=None, maximize=False):
    """value and d/dx of acq_oracle's `kind` at one test point (partials w.r.t. the moments, then the chain rule);
    best_f None is the point's own mean and is differentiated with it"""
    M, V, dM, dV = _moments_grad(mean, var, dmean, dvar, eps)
    s = np.sqrt(V)
    sgn = 1.0 if maximize else -1.0
    db = dM if best_f is None else 0.0
    b = M if best_f is None else best_f
    if kind == "UE":
        return ao.ue(M, V), dV / (2 * s)
    if kind == "UCB":
        beta = 0.25 if param is None else param
        return ao.ucb(M, V, beta, maximize), sgn * dM + 0.5 * np.sqrt(beta / V) * dV
    if kind == "EI":
        u = sgn * (M - b) / s
        val = ao.ei(np.array([M]), np.array([V]), b, maximize)[0]
        # dEI = phi(u) ds + sgn Phi(u) (dM - db)
        return val, ao._pdf(u) * dV / (2 * s) + sgn * ndtr(u) * (dM - db)
    if kind == "POI":
        xi = 0.01 if param is None else param
        u = sgn * (M - b - xi) / s
        val = ao.poi(np.array([M]), np.array([V]), b, xi, maximize)[0]
        du = sgn * (dM - db) / s - u * dV / (2 * V)
        return val, ao._pdf(u) * du
    raise ValueError(kind)
