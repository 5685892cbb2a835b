"""mtgp_grad_oracle.py -- TEST INFRASTRUCTURE ONLY: NumPy restatement of the derivative jax.grad takes through a
MultiTaskGP / CoregGP in the reference's optimize_acq (gpax/acquisition/optimize.py:70-88): the LCM posterior mean and
variance at a test row differentiated w.r.t. that row's inputs.

  kpx_dx           D[p, k, i] = sum_q B_q[t_p, t_i] d k_q(x_p, x_i) / d x_p[k], grad_oracle.kernel_dx per latent on the
                   expanded rows (the Kronecker form's repeated rows each w.r.t. their own point)
  posterior_grad   mean, var (oracle.mtgp_oracle.posterior) and dmean = D alpha, dvar = -2 D K^{-1} k_Xp; the prior
                   diagonal does not depend on x.  In the multitask form the task column comes last with gradient 0:
                   the reference reads it through astype(int) (mtkernels.py:104-105)

Pinned on the CPU by central differences of mtgp_oracle.posterior (tests/test_mtgp_posterior_grad_cpu.py)."""
import numpy as np

from oracle import grad_oracle as gro
from oracle import mtgp_oracle as mo


def task_matrices(params):
    """B_q = W_q W_q^T + diag(v_q) (mtkernels.py:60-63), [L, T, T]"""
    W, v = np.asarray(params["W"], dtype=np.float64), np.asarray(params["v"], dtype=np.float64)
    return np.einsum("qtr,qsr->qts", W, W) + v[:, :, None] * np.eye(W.shape[1])


def kpx_dx(X_new, X_train, params, kernel="RBF", shared=False, num_tasks=None):
    """D [P', d, N'] over the expanded test and training rows"""
    Xn, tn, _ = mo.expand(X_new, shared, num_tasks)
    X, t, _ = mo.expand(X_train, shared, num_tasks)
    Bs = task_matrices(params)
    D = 0.0
    for q in range(mo.num_latents(params)):
        D = D + gro.kernel_dx(Xn, X, mo._latent(params, q), kernel) * Bs[q][np.ix_(tn, t)][:, None, :]
    return D


def posterior_grad(X_train, y_train, X_new, params, kernel="RBF", shared=False, num_tasks=None, noiseless=False, jitter=1e-6):
    """(mean [P'], var [P'], dmean [P', d'], dvar [P', d']) with d' = d (Kronecker form) or d + 1 (multitask form, the task
    column's entries 0)"""
    mean, cov = mo.posterior(X_train, y_train, X_new, params, kernel, shared, num_tasks, noiseless, jitter)
    noise = np.asarray(params["noise"], dtype=np.float64)
    K = mo.lcm_cov(X_train, X_train, params, noise, kernel, shared, num_tasks, jitter)
    k_pX = mo.lcm_cov(X_new, X_train, params, np.zeros_like(noise), kernel, shared, num_tasks, 0.0)
    y = np.asarray(y_train, dtype=np.float64)
    alpha = np.linalg.solve(K, y)
    KinvkXp = np.linalg.solve(K, k_pX.T)                                                  # [N', P']
    D = kpx_dx(X_new, X_train, params, kernel, shared, num_tasks)
    dmean = D @ alpha
    dvar = -2 * np.einsum("pkn,np->pk", D, KinvkXp)
    if not shared:
        dmean, dvar = (np.c_[a, np.zeros(len(a))] for a in (dmean, dvar))
    return mean, np.diag(cov).copy(), dmean, dvar
