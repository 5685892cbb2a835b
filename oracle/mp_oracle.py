"""mp_oracle.py -- the exact-GP posterior in 60-digit arithmetic (mpmath) for small N.  TEST INFRASTRUCTURE ONLY.

SURVEY.md 8c asks for an arbiter: the reference inverts K explicitly in floating point (gpax/models/gp.py:271), so the
fp64 restatement of it (gp_oracle.exact_posterior) carries an error of order cond(K) * eps of its own.  When the CUDA
path and that oracle disagree near the tolerance, this module says which of them is closer to the mathematical
posterior the reference formulates:
    mean = k_pX K^-1 y ,   cov = k_pp - k_pX K^-1 k_Xp          (gp.py:267-273, same Gram rules: kernels.py:44-117)
Only tests/ may import it."""
import mpmath as mp
import numpy as np

mp.mp.dps = 60


def _mpf(v):
    """an input coordinate as an mpf: float inputs exactly, mpf entries (of an object array) as they are"""
    return v if isinstance(v, mp.mpf) else mp.mpf(float(v))


def _gram(kind, X, Z, ell, scale, period, diag):
    n, m, d = X.shape[0], Z.shape[0], X.shape[1]
    K = mp.matrix(n, m)
    for i in range(n):
        for j in range(m):
            if kind == "Periodic":                                  # kernels.py:94-117
                s = mp.mpf(0)
                for k in range(d):
                    s += (mp.sin(mp.pi * (_mpf(X[i, k]) - _mpf(Z[j, k])) / period) / ell[k]) ** 2
                v = scale * mp.exp(-2 * s)
            else:
                r2 = mp.mpf(0)
                for k in range(d):
                    r2 += ((_mpf(X[i, k]) - _mpf(Z[j, k])) / ell[k]) ** 2
                if kind == "RBF":                                   # kernels.py:44-65
                    v = scale * mp.exp(-r2 / 2)
                else:                                               # Matern-5/2, kernels.py:68-91 (r from r2 + 1e-12)
                    r = mp.sqrt(r2 + mp.mpf("1e-12"))
                    v = scale * (1 + mp.sqrt(5) * r + mp.mpf(5) / 3 * r2) * mp.exp(-mp.sqrt(5) * r)
            K[i, j] = v
    if diag is not None:
        for i in range(min(n, m)):
            K[i, i] += diag
    return K


def exact_posterior_mp(X_train, y_train, X_new, params, kernel="RBF", noiseless=False, jitter=1e-6):
    """(mean [P], cov [P, P]) as float64 arrays rounded from 60-digit results; arguments as gp_oracle.exact_posterior."""
    X = np.asarray(X_train, dtype=np.float64)
    Xn = np.asarray(X_new, dtype=np.float64)
    X = X[:, None] if X.ndim == 1 else X
    Xn = Xn[:, None] if Xn.ndim == 1 else Xn
    d = X.shape[1]
    ell = [mp.mpf(float(v)) for v in np.broadcast_to(np.asarray(params["k_length"], dtype=np.float64).ravel(), (d,))]
    scale = mp.mpf(float(params["k_scale"]))
    noise = mp.mpf(float(params["noise"]))
    period = mp.mpf(float(params.get("period", 1.0)))
    jit = mp.mpf(float(jitter))
    noise_p = mp.mpf(0) if noiseless else noise
    Kxx = _gram(kernel, X, X, ell, scale, period, noise + jit)
    Kpx = _gram(kernel, Xn, X, ell, scale, period, None)
    Kpp = _gram(kernel, Xn, Xn, ell, scale, period, noise_p + jit)
    y = mp.matrix([mp.mpf(float(v)) for v in np.asarray(y_train, dtype=np.float64).ravel()])
    L = mp.cholesky(Kxx)
    alpha = mp.cholesky_solve(Kxx, y)                                # K^-1 y
    mean = Kpx * alpha
    P = Xn.shape[0]
    V = mp.matrix(X.shape[0], P)                                     # L^-1 k_Xp, column by column
    for p in range(P):
        col = mp.lu_solve(L, Kpx[p, :].T)
        for i in range(X.shape[0]):
            V[i, p] = col[i]
    cov = Kpp - V.T * V
    return (np.array([float(mean[i]) for i in range(P)]), np.array([[float(cov[i, j]) for j in range(P)] for i in range(P)]))
