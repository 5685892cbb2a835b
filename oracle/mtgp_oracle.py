"""mtgp_oracle.py -- NumPy restatement of MultiTaskGP / CoregGP (gpax/models/mtgp.py, corgp.py).  TEST INFRASTRUCTURE ONLY.

  lcm_cov            the LCM kernel of mtkernels.py:197-233, built from variants_oracle's multitask_kernel (multitask form)
                     or multivariate_kernel (Kronecker form), one per latent, summed
  posterior          gp.py:253-277 with that kernel: the explicit inverse of k_XX
  loglik             log N(y; 0, K) by Cholesky (the likelihood of mtgp.py:162-167 / corgp.py:93-98)
  loglik_grad        its analytic gradient: dK built explicitly for every parameter on the expanded rows (small N)

One draw's parameters: k_length [L, d], k_scale [L], period [L] (Periodic) or None, W [L, T, R], v [L, T], noise [T].
Gradients: w.r.t. log k_length, log k_scale, log period ([L, d+2]), B_q with independent entries ([L, T, T]), log noise [T]."""
import numpy as np
import scipy.linalg as sla

from . import gp_oracle as go
from . import variants_oracle as vo


def _latent(params, q):
    return {k: (None if v is None else np.asarray(v)[q]) for k, v in params.items() if k != "noise"}


def num_latents(params):
    return len(np.asarray(params["k_scale"]).reshape(-1))


def lcm_cov(X, Z, params, noise, kernel="RBF", shared=False, num_tasks=None, jitter=1e-6):
    """mtkernels.py:226-230: sum over latents of the multi-task (shared=False: task id in the last column of X, Z) or
    Kronecker (shared=True: rows point-major, task index fastest) kernel"""
    out = 0.0
    for q in range(num_latents(params)):
        pq = _latent(params, q)
        if shared:
            out = out + vo.multivariate_kernel(X, Z, pq, noise, kernel, num_tasks, jitter)
        else:
            out = out + vo.multitask_kernel(X, Z, pq, noise, kernel, jitter)
    return out


def posterior(X_train, y_train, X_new, params, kernel="RBF", shared=False, num_tasks=None, noiseless=False, jitter=1e-6):
    """gp.py:253-277 (mean, cov) with the LCM kernel"""
    noise = np.asarray(params["noise"])
    noise_p = noise * (1 - int(bool(noiseless)))
    k_pp = lcm_cov(X_new, X_new, params, noise_p, kernel, shared, num_tasks, jitter)
    k_pX = lcm_cov(X_new, X_train, params, np.zeros_like(noise), kernel, shared, num_tasks, 0.0)
    k_XX = lcm_cov(X_train, X_train, params, noise, kernel, shared, num_tasks, jitter)
    K_xx_inv = np.linalg.inv(k_XX)
    cov = k_pp - k_pX @ (K_xx_inv @ k_pX.T)
    mean = k_pX @ (K_xx_inv @ y_train)
    return mean, cov


def loglik(X, y, params, kernel="RBF", shared=False, num_tasks=None, jitter=1e-6):
    K = lcm_cov(X, X, params, np.asarray(params["noise"]), kernel, shared, num_tasks, jitter)
    Lc = sla.cholesky(K, lower=True)
    a = sla.solve_triangular(Lc, y, lower=True)
    return -0.5 * a @ a - np.log(np.diag(Lc)).sum() - 0.5 * len(y) * np.log(2 * np.pi)


def expand(X, shared, num_tasks):
    """(data rows [n, d], task ids [n], group): the Kronecker form repeats each point once per task"""
    X = np.asarray(X, dtype=np.float64)
    if shared:
        T = int(num_tasks)
        return np.repeat(X, T, axis=0), np.tile(np.arange(T), X.shape[0]), T
    return X[:, :-1], X[:, -1].astype(int), 1


def _data_kernel_and_derivs(Xr, pq, kernel):
    """k [n, n] of one latent (no diagonal term) and dk/dlog(ell_k) for every k, dk/dlog(scale), dk/dlog(period)"""
    ell = np.broadcast_to(np.asarray(pq["k_length"], dtype=np.float64).reshape(-1), (Xr.shape[1],))
    s = float(pq["k_scale"])
    diff = Xr[:, None, :] - Xr[None, :, :]
    if kernel == "Periodic":
        p = float(pq["period"])
        a = np.pi * diff / p
        qk = np.sin(a) ** 2 / ell ** 2
        k = s * np.exp(-2 * qk.sum(-1))
        dl = [k * 4 * qk[..., i] for i in range(Xr.shape[1])]
        dp = k * 4 * (np.sin(a) * np.cos(a) * a / ell ** 2).sum(-1)
        return k, dl, k, dp
    qk = (diff / ell) ** 2
    r2 = qk.sum(-1)
    if kernel == "RBF":
        k = s * np.exp(-0.5 * r2)
        dK = k
    else:
        r = np.sqrt(r2 + 1e-12)
        k = s * (1 + np.sqrt(5) * r + 5 / 3 * r2) * np.exp(-np.sqrt(5) * r)
        dK = 5 / 3 * s * (1 + np.sqrt(5) * r) * np.exp(-np.sqrt(5) * r)
    return k, [dK * qk[..., i] for i in range(Xr.shape[1])], k, np.zeros_like(k)


def loglik_grad(X, y, params, kernel="RBF", shared=False, num_tasks=None, jitter=1e-6):
    """(value, g_theta [L, d+2], g_B [L, T, T], g_noise [T]) with value = loglik and the gradient
    1/2 tr((alpha alpha^T - K^{-1}) dK) for each parameter, dK formed explicitly on the expanded rows"""
    Xr, t, group = expand(X, shared, num_tasks)
    n, d = Xr.shape
    Lq = num_latents(params)
    W, v = np.asarray(params["W"], dtype=np.float64), np.asarray(params["v"], dtype=np.float64)
    Bs = np.einsum("qtr,qsr->qts", W, W) + np.stack([np.diag(v[q]) for q in range(Lq)])
    noise = np.asarray(params["noise"], dtype=np.float64)
    T = Bs.shape[1]
    same = (np.arange(n)[:, None] // group) == (np.arange(n)[None, :] // group)
    K = np.zeros((n, n))
    parts = []
    for q in range(Lq):
        k, dl, ds, dp = _data_kernel_and_derivs(Xr, _latent(params, q), kernel)
        Bt = Bs[q][np.ix_(t, t)]
        K += (k + jitter * same) * Bt
        parts.append((k + jitter * same, Bt, dl, ds, dp))
    K[np.diag_indices(n)] += Lq * (noise[t] + jitter)
    Kinv = np.linalg.inv(K)
    alpha = Kinv @ y
    Wm = np.outer(alpha, alpha) - Kinv
    value = loglik(X, y, params, kernel, shared, num_tasks, jitter)
    g_th, g_B = np.zeros((Lq, d + 2)), np.zeros((Lq, T, T))
    for q, (kj, Bt, dl, ds, dp) in enumerate(parts):
        for i in range(d):
            g_th[q, i] = 0.5 * np.sum(Wm * dl[i] * Bt)
        g_th[q, d] = 0.5 * np.sum(Wm * ds * Bt)
        g_th[q, d + 1] = 0.5 * np.sum(Wm * dp * Bt)
        for a in range(T):
            for b in range(T):
                g_B[q, a, b] = 0.5 * np.sum((Wm * kj)[np.ix_(t == a, t == b)])
    g_n = np.array([0.5 * np.sum(np.diag(Wm)[t == a]) * Lq * noise[a] for a in range(T)])
    return value, g_th, g_B, g_n
