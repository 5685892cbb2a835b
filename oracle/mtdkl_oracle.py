"""mtdkl_oracle.py -- NumPy restatement of multi-task deep kernel learning (gpax/models/vi_mtdkl.py).  TEST INFRASTRUCTURE
ONLY (see oracle/__init__.py).

  lcm_dz        log N(y; 0, K(z)) with the LCM covariance (mtgp_oracle.loglik_grad) and d/dz in closed form:
                g_i = sum_{j != i} W_ij sum_q B_q[t_i, t_j] dk_q(z_i, z_j)/dz_i, W = alpha alpha^T - K^-1, on the GP rows;
                the gradient of a point is the sum of its `group` rows
  mtdkl_mll     the same on z = MLP(X) (dkl_oracle.mlp_forward), with the backward pass (dkl_oracle.backward)
  vimtdkl_loss  the Trace_ELBO loss of viMTDKL with AutoDelta for a vector u of the kernel sites (log k_length [L, d],
                k_scale [L], W [L, T, R], log v [L, T], log noise [T]) and the flat network, priors in the constrained space
                without the Jacobian; its gradient
  posterior     the LCM posterior on the embeddings (mtgp_oracle.posterior)

One draw's kernel parameters: k_length [L, d], k_scale [L], W [L, T, R], v [L, T], noise [T].  Multitask form: task ids
given per point (group = 1); Kronecker form: every point observed for every task, rows point-major (group = T)."""
import math

import numpy as np

from . import dkl_oracle as dko
from . import grad_oracle as gro
from . import mtgp_oracle as mo


def _gp_inputs(Z, task, shared, T):
    """the X of mtgp_oracle: z with the task column (multitask form) or the points (Kronecker form)"""
    return np.asarray(Z, dtype=np.float64) if shared else np.column_stack([Z, task])


def lcm_dz(kind, Z, task, y, params, shared, T, jitter=1e-6):
    """(value, g_theta [L, d+2], g_B [L, T, T], g_noise [T], grad_z [n, d] per point, scale_z) for embeddings Z [n, d]"""
    Z = np.asarray(Z, dtype=np.float64)
    X = _gp_inputs(Z, task, shared, T)
    value, g_th, g_B, g_n = mo.loglik_grad(X, y, params, kind, shared, T, jitter)
    Zr, t, group = mo.expand(X, shared, T)
    n, d = Zr.shape
    Lq = mo.num_latents(params)
    W, v = np.asarray(params["W"], dtype=np.float64), np.asarray(params["v"], dtype=np.float64)
    Bs = np.einsum("qtr,qsr->qts", W, W) + np.stack([np.diag(v[q]) for q in range(Lq)])
    K = mo.lcm_cov(X, X, params, np.asarray(params["noise"]), kind, shared, T, jitter)
    Kinv = np.linalg.inv(K)
    Kinv = (Kinv + Kinv.T) / 2
    alpha = Kinv @ y
    aa = np.outer(alpha, alpha)
    Wm = aa - Kinv
    np.fill_diagonal(Wm, 0.0)
    gz, sz = np.zeros((n, d)), np.zeros((n, d))
    for q in range(Lq):
        pq = {"k_length": np.asarray(params["k_length"])[q], "k_scale": float(np.asarray(params["k_scale"]).reshape(-1)[q]),
              "noise": 0.0}
        Dk = gro.kernel_dx(Zr, Zr, pq, kind) * Bs[q][np.ix_(t, t)][:, None, :]      # [n, d, n]
        gz += np.einsum("ij,ikj->ik", Wm, Dk)
        sz += np.einsum("ij,ikj->ik", np.abs(aa) + np.abs(Kinv), np.abs(Dk))
    return value, g_th, g_B, g_n, gz.reshape(-1, group, d).sum(1), sz.reshape(-1, group, d).sum(1)


def mtdkl_mll(kind, X, task, y, layers, act, params, shared, T, jitter=1e-6):
    """(value, g_theta, g_B, g_noise, grad_params (flat), grad_z, scale_z) of the LCM likelihood on z = MLP(X)"""
    H = dko.mlp_forward(X, layers, act)
    value, g_th, g_B, g_n, gz, sz = lcm_dz(kind, H[-1], task, y, params, shared, T, jitter)
    return value, g_th, g_B, g_n, dko.backward(H, layers, act, gz), gz, sz


def sites_from_u(u, L, T, R, d):
    """the kernel-site vector u -> params (constrained)"""
    o = 0

    def take(n):
        nonlocal o
        o += n
        return u[o - n:o]
    ell = np.exp(take(L * d)).reshape(L, d)
    scale = take(L).copy()
    W = take(L * T * R).reshape(L, T, R)
    v = np.exp(take(L * T)).reshape(L, T)
    noise = np.exp(take(T))
    return {"k_length": ell, "k_scale": scale, "W": W, "v": v, "noise": noise}


def _lognormal(t):
    return -np.log(t) - 0.5 * math.log(2 * math.pi) - 0.5 * np.log(t) ** 2


def vimtdkl_loss(kind, X, task, y, u, flat, D, widths, act, L, T, R, shared, jitter=1e-6, nn_prior=True):
    """(loss, grad) over (u, flat) with the default priors: LogNormal(0, 1) k_length, v, noise; Normal(1, 1e-4) k_scale;
    Normal(0, 10) W; Normal(0, 1) weights and Cauchy(0, 1) biases"""
    d = widths[-1] if widths else D
    p = sites_from_u(u, L, T, R, d)
    layers = dko.unflatten(flat, D, widths)
    value, g_th, g_B, g_n, gp, _, _ = mtdkl_mll(kind, X, task, y, layers, act, p, shared, T, jitter)
    s = p["k_scale"]
    val = value + _lognormal(p["k_length"]).sum() + _lognormal(p["v"]).sum() + _lognormal(p["noise"]).sum()
    val += (-0.5 * ((s - 1.0) / 1e-4) ** 2 - math.log(1e-4) - 0.5 * math.log(2 * math.pi)).sum()
    val += (-0.5 * (p["W"] / 10.0) ** 2 - math.log(10.0) - 0.5 * math.log(2 * math.pi)).sum()
    # d/du: log-sites take the likelihood's d/dlog directly plus the LogNormal prior's -1 - log t
    g_ell = g_th[:, :d] - 1.0 - np.log(p["k_length"])
    g_s = g_th[:, d] / s - (s - 1.0) / 1e-8
    g_W = np.einsum("qab,qbr->qar", g_B + g_B.transpose(0, 2, 1), p["W"]) - p["W"] / 100.0
    g_v = np.diagonal(g_B, axis1=1, axis2=2) * p["v"] - 1.0 - np.log(p["v"])
    g_nz = g_n - 1.0 - np.log(p["noise"])
    if nn_prior:
        for W, b in layers:
            val += (-0.5 * W ** 2 - 0.5 * math.log(2 * math.pi)).sum() + (-math.log(math.pi) - np.log1p(b ** 2)).sum()
        gp = gp + dko.flatten([(-W, -2.0 * b / (1.0 + b ** 2)) for W, b in layers])
    g = np.concatenate([g_ell.ravel(), g_s, g_W.ravel(), g_v.ravel(), g_nz, gp])
    return -val, -g


def posterior(kind, X, task, y, X_new, task_new, layers, act, params, shared, T, noiseless=False, jitter=1e-6):
    """(mean, cov) of the LCM GP on the embeddings (vi_mtdkl.py:211-247)"""
    z = dko.mlp_forward(X, layers, act)[-1]
    zn = dko.mlp_forward(X_new, layers, act)[-1]
    return mo.posterior(_gp_inputs(z, task, shared, T), y, _gp_inputs(zn, task_new, shared, T), params, kind, shared, T,
                        noiseless, jitter)
