"""ibnn_oracle.py -- NumPy restatement of iBNN / vi_iBNN (gpax/models/ibnn.py, gpax/models/vi_ibnn.py).  TEST
INFRASTRUCTURE ONLY (see oracle/__init__.py).

  kernel       the NNGP Gram matrix (variants_oracle.nngp_kernel, gpax/kernels/kernels.py:120-224)
  kernel_grad  the Gram matrix and its derivatives w.r.t. var_b and var_w, in closed forward mode as JAX differentiates
               the reference: zero through jnp.clip where the clip is active, the unclipped fraction entering the ReLU
               step through (pi - theta) * fraction, both square roots differentiated through both arguments
  mll          log N(y; 0, K) by a SciPy Cholesky factor
  mll_grad     its value and gradient w.r.t. (log var_w, log noise, log var_b): 1/2 tr((alpha alpha^T - K^-1) dK)
  posterior    the ExactGP posterior on the NNGP kernel (gp_oracle.exact_posterior, gp.py:253-277)
  vi_predict   viGP.predict on it (vigp.py:178-185)

params: {"var_b", "var_w", "noise"}; activation 'erf' or 'relu'."""
import math

import numpy as np
import scipy.linalg as sla

from . import gp_oracle as go
from . import variants_oracle as vo


def kernel(X, Z, params, noise=0, jitter=1e-6, activation="erf", depth=3):
    return vo.nngp_kernel(go._as2d(X), go._as2d(Z), params, noise, jitter, activation, depth)


def _step(act, a, b, c, vb, vw):
    """one layer on (value, d/dvar_b, d/dvar_w) triples a = k12, b = k11, c = k22"""
    (a0, ab, aw), (b0, bb, bw), (c0, cb, cw) = a, b, c
    if act == "erf":
        u = (1 + 2 * b0) * (1 + 2 * c0)
        s = np.sqrt(u)
        fr = 2 * a0 / s
        frc = np.clip(fr, -1 + 1e-7, 1 - 1e-7)
        th = np.arcsin(frc)
        live = (fr == frc)
        k = np.where(live, 2 * vw / np.pi / np.sqrt(1 - frc * frc), 0.0)
        dfr = [2 * da / s - fr / (2 * u) * (2 * db * (1 + 2 * c0) + 2 * dc * (1 + 2 * b0))
               for da, db, dc in ((ab, bb, cb), (aw, bw, cw))]
        return vb + 2 * vw / np.pi * th, 1 + k * dfr[0], 2 / np.pi * th + k * dfr[1]
    s = np.sqrt(b0 * c0)
    fr = a0 / s
    frc = np.clip(fr, -1 + 1e-7, 1 - 1e-7)
    th = np.arccos(frc)
    live = (fr == frc)
    t = np.sin(th) + (np.pi - th) * fr
    out = [vb + vw / (2 * np.pi) * s * t]
    for p, (da, db, dc) in enumerate(((ab, bb, cb), (aw, bw, cw))):
        ds = (db * c0 + b0 * dc) / (2 * s)
        dfr = da / s - a0 * ds / s ** 2
        dth = np.where(live, -dfr / np.sqrt(1 - frc * frc), 0.0)
        dt = np.cos(th) * dth - fr * dth + (np.pi - th) * dfr
        out.append((1.0 if p == 0 else 0.0) + vw / (2 * np.pi) * (ds * t + s * dt) + (s * t / (2 * np.pi) if p == 1 else 0.0))
    return tuple(out)


def kernel_grad(X, Z, var_b, var_w, activation="erf", depth=3):
    """(K, dK/dvar_b, dK/dvar_w) of the NNGP kernel without the diagonal term"""
    X, Z = go._as2d(X), go._as2d(Z)
    d = X.shape[1]
    xz = X @ Z.T
    xx = (X * X).sum(1)[:, None] * np.ones((1, Z.shape[0]))
    zz = np.ones((X.shape[0], 1)) * (Z * Z).sum(1)[None, :]
    one = np.ones_like(xz)
    k12, k11, k22 = ((var_b + var_w * v / d, one, v / d) for v in (xz, xx, zz))      # depth 0, kernels.py:139-140
    for _ in range(depth):
        k12, k11, k22 = (_step(activation, k12, k11, k22, var_b, var_w), _step(activation, k11, k11, k11, var_b, var_w),
                         _step(activation, k22, k22, k22, var_b, var_w))
    return k12


def mll(X, y, params, activation="erf", depth=3, jitter=1e-6):
    K = kernel(X, X, params, params["noise"], jitter, activation, depth)
    L = sla.cholesky(K, lower=True)
    w = sla.solve_triangular(L, np.asarray(y, dtype=np.float64), lower=True)
    return -0.5 * w @ w - np.log(np.diag(L)).sum() - 0.5 * len(w) * math.log(2 * math.pi)


def mll_grad(X, y, params, activation="erf", depth=3, jitter=1e-6, noise_vec=None):
    """(value, [d/dlog var_w, d/dlog noise, d/dlog var_b]); noise_vec: per-point noise variances added to the diagonal"""
    vb, vw, noise = float(params["var_b"]), float(params["var_w"]), float(params["noise"])
    Kf, dKb, dKw = kernel_grad(X, X, vb, vw, activation, depth)
    K = Kf + (noise + jitter) * np.eye(Kf.shape[0])
    if noise_vec is not None:
        K = K + np.diag(noise_vec)
    cf = sla.cho_factor(K, lower=True)
    y = np.asarray(y, dtype=np.float64)
    alpha = sla.cho_solve(cf, y)
    Kinv = sla.cho_solve(cf, np.eye(K.shape[0]))
    W = np.outer(alpha, alpha) - Kinv
    value = -0.5 * y @ alpha - np.log(np.diag(cf[0])).sum() - 0.5 * len(y) * math.log(2 * math.pi)
    g = np.array([0.5 * np.sum(W * dKw) * vw, 0.5 * np.trace(W) * noise, 0.5 * np.sum(W * dKb) * vb])
    return value, g


def posterior(X_train, y_train, X_new, params, activation="erf", depth=3, noiseless=False, **kwargs):
    kern = lambda X, Z, p, noise=0, jitter=1e-6: kernel(X, Z, p, noise, jitter, activation, depth)   # noqa: E731
    return go.exact_posterior(X_train, y_train, X_new, params, kern, noiseless, **kwargs)


def vi_predict(X_train, y_train, X_new, params, activation="erf", depth=3, noiseless=False, **kwargs):
    mean, cov = posterior(X_train, y_train, X_new, params, activation, depth, noiseless, **kwargs)
    return mean, np.diag(cov)
