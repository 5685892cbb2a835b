"""NumPy fp64 restatement of the sparse GP from caller-supplied Gram blocks (b2gp_sparse_elbo_gram,
b2gp_sparse_posterior_gram), derived without the library's reverse pass.

The bound, with Ks = (Kuu + Kuu^T) / 2, V = Ks^-1 Kuf, Q = Kuf^T V and S = Q + noise I:
    value = log N(y; 0, S) - 1/2 max(T, 0) / noise,   T = sum kff_diag - tr(Q)
With alpha = S^-1 y and B = 1/2 (alpha alpha^T - S^-1) + coef / (2 noise) I (coef = 1 while T > 0), the first-order
change is tr(B dQ) - coef / (2 noise) sum dkff, and dQ = dKuf^T V + V^T dKuf - V^T dKs V gives the adjoints
    Guf = 2 V B,   Gs = -V B V^T   (symmetric, so sum Gs * dKuu = sum Gs * dKs for any dKuu),
and d value / d noise = 1/2 tr(alpha alpha^T - S^-1) + coef T / (2 noise^2).
"""
import numpy as np
import scipy.linalg as sla

LOG2PI = 1.8378770664093453


def elbo_gram_grad(Kuu, Kuf, kff_diag, y, noise, dirs=(), rdirs=()):
    """(value, grad [len(dirs)], grad_log_noise, grad_rows [len(rdirs), M], alpha [N]) for directions (dKuu, dKuf, dkff)
    and row directions (rKuu, rKuf); None blocks are zero"""
    Kuu, Kuf, y = np.asarray(Kuu, float), np.asarray(Kuf, float), np.asarray(y, float)
    M, N = Kuf.shape
    Ks = (Kuu + Kuu.T) / 2
    Lu = sla.cholesky(Ks, lower=True)
    V = sla.cho_solve((Lu, True), Kuf)
    Q = Kuf.T @ V
    Q = (Q + Q.T) / 2
    T = float(np.sum(kff_diag)) - np.trace(Q)
    coef = 1.0 if T > 0 else 0.0
    S = Q + noise * np.eye(N)
    Ls = sla.cholesky(S, lower=True)
    alpha = sla.cho_solve((Ls, True), y)
    Sinv = sla.cho_solve((Ls, True), np.eye(N))
    value = -0.5 * y @ alpha - np.log(np.diag(Ls)).sum() - 0.5 * N * LOG2PI - (0.5 * T / noise if T > 0 else 0.0)
    A = np.outer(alpha, alpha) - Sinv
    B = 0.5 * A + coef / (2 * noise) * np.eye(N)
    Guf = 2 * V @ B
    Gs = -V @ B @ V.T
    Gs = (Gs + Gs.T) / 2
    gd = -coef / (2 * noise)
    grad = np.array([(0.0 if du is None else np.sum(Gs * du)) + (0.0 if df is None else np.sum(Guf * df))
                     + (0.0 if dk is None else gd * np.sum(dk)) for du, df, dk in dirs])
    rows = np.array([(0.0 if ru is None else np.sum(Gs * ru, axis=1)) + (0.0 if rf is None else np.sum(Guf * rf, axis=1))
                     + np.zeros(M) for ru, rf in rdirs]).reshape(len(rdirs), M)
    gnoise = 0.5 * np.trace(A) + coef * T / (2 * noise ** 2)
    return value, grad, noise * gnoise, rows, alpha


def sparse_posterior_gram(Kuu, Kuf, y, noise, Kus, Kss):
    """(mean [P], cov [P, P]) of gpax/models/sparse_gp.py:189-217 from the blocks (Kss holds noise_p already)"""
    Luu = sla.cholesky(np.asarray(Kuu, float), lower=True)
    W = sla.solve_triangular(Luu, Kuf, lower=True)
    K = (W / noise) @ W.T + np.eye(W.shape[0])
    L = sla.cholesky(K, lower=True)
    Ws = sla.solve_triangular(Luu, Kus, lower=True)
    pack = sla.solve_triangular(L, np.column_stack([(W / noise) @ y, Ws]), lower=True)
    mean = pack[:, 0] @ pack[:, 1:]
    cov = Kss - Ws.T @ Ws + pack[:, 1:].T @ pack[:, 1:]
    return mean, cov
