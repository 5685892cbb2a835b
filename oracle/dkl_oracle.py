"""dkl_oracle.py -- NumPy restatement of deep kernel learning (gpax/models/vidkl.py, gpax/models/dkl.py).  TEST
INFRASTRUCTURE ONLY (see oracle/__init__.py).

  mlp_forward      H_{l+1} = act(H_l W_l + b_l), no activation after the last layer (vidkl.py:400-412, dkl.py:167-177)
  mll_dz           log N(y; 0, K(z)), d/dlog theta (fit_oracle.mll_grad) and d/dz_i = sum_j W_ij dk(z_i, z_j)/dz_i with
                   W = alpha alpha^T - K^-1 and grad_oracle.kernel_dx's derivatives
  dkl_mll          the same on z = MLP(X), with the backward pass to every weight and bias
  vidkl_loss       the Trace_ELBO loss of viDKL with AutoDelta: -(mll + sum log N(w) + sum log Cauchy(b) + sum log p(theta)),
                   theta's priors in the constrained space without the Jacobian; its gradient w.r.t. (log theta, weights)
  adam             Adam(b1 = 0.5) as numpyro.optim.Adam
  posterior        the exact posterior on embeddings (gp_oracle.exact_posterior)

Layers are lists of (W [in, out], b [out]); theta is [lengthscale[d], k_scale, noise, period]; act 'relu' or 'tanh'."""
import math

import numpy as np

from . import fit_oracle as fo
from . import gp_oracle as go
from . import grad_oracle as gro


def _act(h, act):
    return np.maximum(h, 0.0) if act == "relu" else np.tanh(h)


def _act_grad(h, act):
    return (h > 0).astype(np.float64) if act == "relu" else 1.0 - h * h


def flatten(layers):
    return np.concatenate([np.concatenate([np.asarray(W).ravel(), np.asarray(b).ravel()]) for W, b in layers])


def unflatten(flat, D, widths):
    out, o, i = [], 0, D
    for w in widths:
        W = flat[o:o + i * w].reshape(i, w)
        o += i * w
        out.append((W, flat[o:o + w]))
        o += w
        i = w
    return out


def mlp_forward(X, layers, act):
    """activations [X, H_1, ..., z]"""
    H = [np.asarray(X, dtype=np.float64)]
    for l, (W, b) in enumerate(layers):
        h = H[-1] @ W + b
        H.append(_act(h, act) if l + 1 < len(layers) else h)
    return H


def mll_dz(kind, Z, y, theta, jitter):
    """(value, grad_theta [d+3], grad_z [N, d], scale_z [N, d]): scale_z is the size of the terms summed into each entry"""
    Z = np.asarray(Z, dtype=np.float64)
    N, d = Z.shape
    value, g, alpha, _, _ = fo.mll_grad(kind, Z, y, theta, jitter)
    k, _ = fo._derivs(Z, theta, kind)
    K = k.copy()
    K[np.diag_indices(N)] += theta[d + 1] + jitter
    Kinv = np.linalg.inv(K)
    Kinv = (Kinv + Kinv.T) / 2
    aa = np.outer(alpha, alpha)
    Wm = aa - Kinv
    np.fill_diagonal(Wm, 0.0)
    Dk = gro.kernel_dx(Z, Z, {**fo._params(theta, d), "noise": theta[d + 1]}, kind)     # [N, d, N]
    gz = np.einsum("ij,ikj->ik", Wm, Dk)
    sz = np.einsum("ij,ikj->ik", np.abs(aa) + np.abs(Kinv), np.abs(Dk))
    return value, g, gz, sz


def backward(H, layers, act, gz):
    """d/d(W_l, b_l) from d/dz, in the flat layout"""
    G, grads = gz, [None] * len(layers)
    for l in range(len(layers) - 1, -1, -1):
        W, _ = layers[l]
        grads[l] = (H[l].T @ G, G.sum(0))
        if l > 0:
            G = (G @ W.T) * _act_grad(H[l], act)
    return flatten(grads) if grads else np.zeros(0)


def dkl_mll(kind, X, y, layers, act, theta, jitter):
    """(value, grad_theta, grad_params (flat), grad_z, scale_z) of log N(y; 0, K(MLP(X)))"""
    H = mlp_forward(X, layers, act)
    value, g, gz, sz = mll_dz(kind, H[-1], y, theta, jitter)
    return value, g, backward(H, layers, act, gz), gz, sz


def _theta_sites(kind, d):
    """(positions in theta) of the LogNormal(0, 1) kernel and noise sites (gp.py:222-247)"""
    return list(range(d + 2)) + ([d + 2] if kind == "Periodic" else [])


def vidkl_loss(kind, X, y, u_theta, flat, D, widths, act, jitter, nn_prior=True):
    """(loss, grad) over (u_theta = log theta at the sampled sites, flat network parameters)"""
    d = widths[-1]
    idx = _theta_sites(kind, d)
    theta = np.ones(d + 3)
    theta[idx] = np.exp(u_theta)
    layers = unflatten(flat, D, widths)
    value, g, gp, _, _ = dkl_mll(kind, X, y, layers, act, theta, jitter)
    t = theta[idx]
    lp = -np.log(t) - 0.5 * math.log(2 * math.pi) - 0.5 * np.log(t) ** 2           # LogNormal(0, 1)
    gu = g[idx] + (-1.0 / t - np.log(t) / t) * t
    val = value + lp.sum()
    if nn_prior:
        for W, b in layers:
            val += (-0.5 * W ** 2 - 0.5 * math.log(2 * math.pi)).sum() + (-math.log(math.pi) - np.log1p(b ** 2)).sum()
        prior_g = flatten([(-W, -2.0 * b / (1.0 + b ** 2)) for W, b in layers])
        gp = gp + prior_g
    return -val, -np.concatenate([gu, gp])


def adam(loss_grad, params, num_steps, step_size):
    """numpyro.optim.Adam(step_size, b1=0.5): losses per step and the final parameters"""
    m1, m2 = np.zeros_like(params), np.zeros_like(params)
    b1, b2, eps = 0.5, 0.999, 1e-8
    losses = []
    for t in range(1, num_steps + 1):
        loss, g = loss_grad(params)
        losses.append(loss)
        m1 = b1 * m1 + (1 - b1) * g
        m2 = b2 * m2 + (1 - b2) * g * g
        params = params - step_size * (m1 / (1 - b1 ** t)) / (np.sqrt(m2 / (1 - b2 ** t)) + eps)
    return np.array(losses), params


def posterior(kind, X, y, X_new, layers, act, params, noiseless=False, jitter=1e-6):
    """(mean, cov) of the exact GP on the embeddings (vidkl.py:206-236, dkl.py:113-132)"""
    z = mlp_forward(X, layers, act)[-1]
    zn = mlp_forward(X_new, layers, act)[-1]
    return go.exact_posterior(z, y, zn, params, kind, noiseless, jitter=jitter)
