"""fit_oracle.py -- closed-form references of the fit-side entry points.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

  mll_grad         b2gp_mll / b2gp_mll_v: value = log N(y; 0, K), its gradient 1/2 sum (alpha alpha^T - K^-1) o dK w.r.t.
                   log(lengthscale[d], k_scale, noise, period), alpha = K^-1 y, d value / d noise_vec, and per entry the
                   size of the terms that cancel in it (`scale`)
  elbo_grad        b2gp_sparse_elbo: the VFE bound of viSparseGP and its gradient w.r.t. log theta and Xu, derived on the
                   dense N x N covariance S = Kfu Kuu^-1 Kuf + noise I (the library works on the M x M Woodbury form, so
                   the two derivations share nothing but the kernel derivatives)
  mll_mp, elbo_mp  the same values in 60-digit arithmetic (mp_oracle._gram); *_grad_mp differentiate them with mp.diff,
                   i.e. central differences carried out in 60 digits (tiny problems: N <= 24, M <= 6)
  tau              the tolerance rule of the GPU tests; `mutate=` of mll_grad / elbo_grad plants one named defect in the
                   reference, which that tolerance must reject

theta follows the C ABI: [lengthscale[d], k_scale, noise, period] in natural units; kernels are "RBF", "Matern",
"Periodic".  dK/dlog(theta) comes from mtgp_oracle._data_kernel_and_derivs, dK/dXu from grad_oracle.kernel_dx."""
import mpmath as mp
import numpy as np
import scipy.linalg as sla
import scipy.sparse.linalg as spla

from . import grad_oracle as gro
from . import mp_oracle as mpo
from . import mtgp_oracle as mto

LOG2PI = float(np.log(2 * np.pi))
MLL_TILE = 64                      # the tile of mll_grad_kernel (csrc/mll.cuh)


def _params(theta, d):
    theta = np.asarray(theta, dtype=np.float64)
    return {"k_length": theta[:d], "k_scale": float(theta[d]), "period": float(theta[d + 2])}


def _derivs(Z, theta, kind):
    """k(Z, Z) without diagonal terms and the d+3 matrices dk/dlog(theta) (the noise slot is None: it is a diagonal)"""
    d = Z.shape[1]
    k, dl, ds, dp = mto._data_kernel_and_derivs(Z, _params(theta, d), kind)
    return k, list(dl) + [ds, None, dp]


# ------------------------------------------------------------------ exact GP likelihood
def mll_grad(kind, X, y, theta, jitter, noise_vec=None, mutate=None):
    """(value, grad [d+3], alpha [N], grad_noise_vec [N] or None, scale [d+3]).  K = k(X, X) + (noise + jitter) I
    (+ diag(noise_vec)); d/dlog(noise) acts on noise alone, not on the jitter.  `mutate` plants a named defect (tests/test_fit_oracle_cpu.py)."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    N, d = X.shape
    noise = float(theta[d + 1])
    k, dK = _derivs(X, theta, kind)
    K = k.copy()
    K[np.diag_indices(N)] += noise + jitter + (0.0 if noise_vec is None else np.asarray(noise_vec, dtype=np.float64))
    Lc = sla.cholesky(K, lower=True)
    w = sla.solve_triangular(Lc, y, lower=True)
    value = -0.5 * w @ w - np.log(np.diag(Lc)).sum() - 0.5 * N * LOG2PI
    alpha = sla.cho_solve((Lc, True), y)
    Kinv = sla.cho_solve((Lc, True), np.eye(N))
    Kinv = (Kinv + Kinv.T) / 2
    if mutate == "kinv_plane":
        # the SYRK K^-1 = B B^T on one digit plane fewer than 7: a six-plane split truncates each operand row at 2^-46 of
        # its norm, and the k = N products of an entry accumulate that like sqrt(k)
        nrm = np.sqrt(np.diag(Kinv))
        Kinv = Kinv + 2.0 ** -46 * np.sqrt(N) * np.outer(nrm, nrm)
    aa = np.outer(alpha, alpha)
    Wm = aa - Kinv
    grad, scale = np.zeros(d + 3), np.zeros(d + 3)
    r0 = MLL_TILE * ((N - 1) // MLL_TILE)
    for p in range(d + 3):
        if dK[p] is None:                      # noise: dK = noise I
            dg = (noise + jitter if mutate == "jitter_noise" else noise) * np.ones(N)
            grad[p] = 0.5 * (np.diag(Wm) * dg).sum()
            scale[p] = 0.5 * ((np.abs(np.diag(aa)) + np.abs(np.diag(Kinv))) * noise).sum()
            D = np.diag(dg)
        else:
            D = dK[p]
            grad[p] = 0.5 * (Wm * D).sum()
            scale[p] = 0.5 * ((np.abs(aa) + np.abs(Kinv)) * np.abs(D)).sum()
        if mutate == "diag2":                  # diagonal entries weighted 2 like the off-diagonal ones
            grad[p] += 0.5 * (np.diag(Wm) * np.diag(D)).sum()
        elif mutate == "drop_tile":            # the last (ragged) diagonal 64-tile never reduced
            grad[p] -= 0.5 * (Wm[r0:, r0:] * D[r0:, r0:]).sum()
    gnv = None if noise_vec is None else 0.5 * (alpha ** 2 - np.diag(Kinv))
    return value, grad, alpha, gnv, scale


# ------------------------------------------------------------------ VFE bound of the sparse GP
def elbo_grad(kind, Xu, X, y, theta, jitter, mutate=None):
    """(value, grad_theta [d+3], grad_Xu [M, d], scale_theta [d+3], scale_Xu [M, d], T) of
        ELBO = log N(y; 0, S) - 1/2 max(T, 0) / noise,   S = Q + noise I,  Q = Kfu Kuu^-1 Kuf,  T = sum_n (Kff_nn - Q_nn)
    with Kuu = k(Xu, Xu) + jitter I and Kuf = k(Xu, X) (no diagonal term).  With A = Kfu Kuu^-1, G = 1/2 (alpha alpha^T -
    S^-1): dELBO/dKuf = 2 A^T G (+ A^T / noise), dELBO/dKuu = -A^T G A (- A^T A / (2 noise)), dELBO/dKff_nn = (-1/(2 noise)),
    the bracketed terms only while the clip is inactive (T > 0)."""
    Xu, X = np.asarray(Xu, dtype=np.float64), np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    M, d = Xu.shape
    N = X.shape[0]
    noise = float(theta[d + 1])
    Z = np.vstack([Xu, X])
    k, dK = _derivs(Z, theta, kind)
    Kuu = k[:M, :M] + jitter * np.eye(M)
    Kuf = k[:M, M:]
    kdiag = np.diag(k)[M:]
    Lu = sla.cholesky(Kuu, lower=True)
    A = sla.cho_solve((Lu, True), Kuf).T                           # N x M
    S = A @ Kuf
    S = (S + S.T) / 2
    T = kdiag.sum() - np.trace(S)
    S[np.diag_indices(N)] += noise
    Ls = sla.cholesky(S, lower=True)
    alpha = sla.cho_solve((Ls, True), y)
    Sinv = sla.cho_solve((Ls, True), np.eye(N))
    Sinv = (Sinv + Sinv.T) / 2
    active = (T > 0) != (mutate == "clip")
    value = -0.5 * y @ alpha - np.log(np.diag(Ls)).sum() - 0.5 * N * LOG2PI - (0.5 * T / noise if T > 0 else 0.0)
    Aa = A.T @ alpha                                               # A^T alpha [M]
    # dELBO/dKuf and dELBO/dKuu as a sum of pieces; |piece| o |dK| summed is the size of what cancels
    uf = [np.outer(Aa, alpha), -(A.T @ Sinv)]                      # 2 A^T G = A^T alpha alpha^T - A^T S^-1
    AtSA = A.T @ Sinv @ A
    uu = [-0.5 * np.outer(Aa, Aa), 0.5 * AtSA]                     # -A^T G A
    if active:
        uf.append(A.T / noise)
        uu.append(-(A.T @ A) / (2 * noise))
    Guf, Guu = sum(uf), sum(uu)
    grad, scale = np.zeros(d + 3), np.zeros(d + 3)
    for p in range(d + 3):
        if dK[p] is None:
            continue
        Duf, Duu = dK[p][:M, M:], dK[p][:M, :M]
        grad[p] = (Guf * Duf).sum() + (Guu * Duu).sum()
        scale[p] = sum((np.abs(P) * np.abs(Duf)).sum() for P in uf) + sum((np.abs(P) * np.abs(Duu)).sum() for P in uu)
    trSinv = np.trace(Sinv)
    grad[d + 1] = noise * (0.5 * alpha @ alpha - 0.5 * trSinv)
    scale[d + 1] = noise * 0.5 * (alpha @ alpha + trSinv)
    if active:                                                     # Kff_nn = k_scale * (kernel at r = 0); T / (2 noise)
        grad[d] -= 0.5 * kdiag.sum() / noise
        scale[d] += 0.5 * kdiag.sum() / noise
        grad[d + 1] += 0.5 * T / noise
        scale[d + 1] += 0.5 * abs(T) / noise
    # Xu[a] moves row a of Kuf and row and column a of Kuu; dK/dXu[a, k] = Dx[a, k, :]
    Dx = gro.kernel_dx(Xu, Z, _params(theta, d), kind)             # [M, d, M + N]
    Dxf, Dxu = Dx[:, :, M:], Dx[:, :, :M]
    gx = np.einsum("an,akn->ak", Guf, Dxf)
    kuu_term = np.einsum("ab,akb->ak", Guu + Guu.T, Dxu)
    if mutate == "xu_kuu":                                         # the Kuu contraction of one inducing point's row lost
        kuu_term[M - 1] = 0.0
    gx = gx + kuu_term
    sx = sum(np.einsum("an,akn->ak", np.abs(P), np.abs(Dxf)) for P in uf)
    sx = sx + sum(np.einsum("ab,akb->ak", np.abs(P) + np.abs(P.T), np.abs(Dxu)) for P in uu)
    return value, grad, gx, scale, sx, T


# ------------------------------------------------------------------ 60-digit arbiter
def _mp_theta(theta):
    return [mp.mpf(float(v)) for v in np.asarray(theta, dtype=np.float64)]


def _mp_logpdf(K, y):
    """log N(y; 0, K) in mpmath"""
    n = K.rows
    L = mp.cholesky(K)
    w = _fwd(L, y)
    return -mp.mpf(1) / 2 * sum(w[i] ** 2 for i in range(n)) - sum(mp.log(L[i, i]) for i in range(n)) - n * mp.log(2 * mp.pi) / 2


def _fwd(L, b):
    """L^-1 b for a lower-triangular mp.matrix L"""
    n = L.rows
    x = [mp.mpf(0)] * n
    for i in range(n):
        s = b[i]
        for j in range(i):
            s -= L[i, j] * x[j]
        x[i] = s / L[i, i]
    return x


def mll_mp(kind, X, y, th, jitter, noise_vec=None):
    """log N(y; 0, K) in 60 digits; th = the d+3 parameters as mpf"""
    d = X.shape[1]
    K = mpo._gram(kind, X, X, th[:d], th[d], th[d + 2], th[d + 1] + mp.mpf(float(jitter)))
    if noise_vec is not None:
        for i in range(X.shape[0]):
            K[i, i] += noise_vec[i]
    return _mp_logpdf(K, [mp.mpf(float(v)) for v in y])


def elbo_mp(kind, Xu, X, y, th, jitter):
    """the VFE bound in 60 digits (Xu may be an object array of mpf)"""
    M, d = Xu.shape
    N = X.shape[0]
    ell, s, noise, per = th[:d], th[d], th[d + 1], th[d + 2]
    Kuu = mpo._gram(kind, Xu, Xu, ell, s, per, mp.mpf(float(jitter)))
    Kuf = mpo._gram(kind, Xu, X, ell, s, per, None)
    kd = mpo._gram(kind, X[:1], X[:1], ell, s, per, None)[0, 0]
    Lu = mp.cholesky(Kuu)
    Wc = [_fwd(Lu, [Kuf[a, n] for a in range(M)]) for n in range(N)]   # column n of W = Luu^-1 Kuf
    S = mp.matrix(N, N)
    for i in range(N):
        for j in range(i + 1):
            S[i, j] = S[j, i] = sum(Wc[i][a] * Wc[j][a] for a in range(M))
    T = N * kd - sum(S[i, i] for i in range(N))
    for i in range(N):
        S[i, i] += noise
    v = _mp_logpdf(S, [mp.mpf(float(t)) for t in y])
    return v - (T / (2 * noise) if T > 0 else 0)


def mll_grad_mp(kind, X, y, theta, jitter, noise_vec=None):
    """(value, d value / dlog(theta) [d+3], d value / d noise_vec or None) from 60-digit values"""
    d = X.shape[1]
    th0 = _mp_theta(theta)
    nv0 = None if noise_vec is None else [mp.mpf(float(v)) for v in noise_vec]

    def at(p):
        return lambda t: mll_mp(kind, X, y, [v * mp.exp(t) if q == p else v for q, v in enumerate(th0)], jitter, nv0)
    g = np.array([float(mp.diff(at(p), 0)) for p in range(d + 3)])
    gnv = None
    if nv0 is not None:
        def at_nv(i):
            return lambda t: mll_mp(kind, X, y, th0, jitter, [v + t if q == i else v for q, v in enumerate(nv0)])
        gnv = np.array([float(mp.diff(at_nv(i), 0)) for i in range(len(nv0))])
    return float(mll_mp(kind, X, y, th0, jitter, nv0)), g, gnv


def elbo_grad_mp(kind, Xu, X, y, theta, jitter):
    """(value, d ELBO / dlog(theta) [d+3], d ELBO / dXu [M, d]) from 60-digit values"""
    M, d = Xu.shape
    th0 = _mp_theta(theta)
    Xu0 = np.array([[mp.mpf(float(v)) for v in row] for row in Xu], dtype=object)

    def at(p):
        return lambda t: elbo_mp(kind, Xu0, X, y, [v * mp.exp(t) if q == p else v for q, v in enumerate(th0)], jitter)

    def at_x(a, k):
        def f(t):
            Z = Xu0.copy()
            Z[a, k] = Z[a, k] + t
            return elbo_mp(kind, Z, X, y, th0, jitter)
        return f
    g = np.array([float(mp.diff(at(p), 0)) for p in range(d + 3)])
    gx = np.array([[float(mp.diff(at_x(a, k), 0)) for k in range(d)] for a in range(M)])
    return float(elbo_mp(kind, Xu0, X, y, th0, jitter)), g, gx


# ------------------------------------------------------------------ tolerances
# fp64 routes: the parity bar of test_gpu_paths.py, 1e-9 at cond <= 1e5 and growing with cond beyond.
# int8 routes: DESIGN 4.6's digit-plane model -- a posterior computed through S digit planes carries an error of about
# cond * C_PLANES[S] -- floored at fp64's unit roundoff (7 planes add less than the fp64 arithmetic around them), times
# INT8_SAFETY.  Each gradient entry is held to tau * (|ref| + scale), scale being the size of the terms that cancel in it.
# The gradients need a larger factor than the posterior: they weigh every entry of K^-1, and the int8 SYRK's error in an
# entry scales with the norms of its two operand rows, not with the entry.  Measured on an H100 SXM (700 W): the largest
# err / tau over tests/test_gpu_fit_paths.py's int8 cases is 0.37 at INT8_SAFETY = 1000 (the N = 600 likelihood whose K^-1
# SYRK alone runs on 7 planes), 0.08 for 6 planes on the tall route.
C_PLANES = {6: 1.3e-16, 7: 3e-18}
EPS64 = 2.0 ** -53
INT8_SAFETY = 1000.0


def tau(cond, planes=0):
    """planes = 0: an fp64 route; 6 or 7: the digit planes of the int8 products on the route"""
    if planes == 0:
        return 1e-9 * max(1.0, cond / 1e5)
    return INT8_SAFETY * max(cond, 1.0) * max(C_PLANES[planes], EPS64)


def err_ratio(got, ref, scale, t):
    """max over entries of |got - ref| / (t (|ref| + scale)): <= 1 passes.  An entry with ref = scale = 0 (the period
    gradient of a non-periodic kernel) must be exactly 0."""
    got, ref, scale = (np.asarray(a, dtype=np.float64) for a in (got, ref, scale))
    num, den = np.abs(got - ref), t * (np.abs(ref) + scale)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(den > 0, num / den, np.where(num > 0, np.inf, 0.0))
    return float(np.max(r)) if r.size else 0.0


def cond_spd(K, lam_min=None):
    """cond(K): lambda_max by Lanczos, lambda_min given (a lower bound such as noise + jitter) or computed"""
    n = K.shape[0]
    if n <= 400 or lam_min is None:
        ev = np.linalg.eigvalsh(K)
        return float(ev[-1] / (ev[0] if lam_min is None else lam_min))
    top = float(spla.eigsh(K, k=1, which="LA", return_eigenvectors=False, tol=1e-4)[0])
    return top / lam_min


def mll_cond(kind, X, theta, jitter, noise_vec=None):
    d = X.shape[1]
    K = mto._data_kernel_and_derivs(X, _params(theta, d), kind)[0]
    floor = theta[d + 1] + jitter + (0.0 if noise_vec is None else float(np.min(noise_vec)))
    K[np.diag_indices(X.shape[0])] += theta[d + 1] + jitter + (0.0 if noise_vec is None else noise_vec)
    return cond_spd(K, floor)


def kuu_cond(kind, Xu, theta, jitter):
    d = Xu.shape[1]
    K = mto._data_kernel_and_derivs(Xu, _params(theta, d), kind)[0] + jitter * np.eye(Xu.shape[0])
    return cond_spd(K)


# ------------------------------------------------------------------ seeded problems shared by the CPU and GPU tests
def mll_problem(kind, N, d, seed, noise=0.1, ell=None, scale=1.3):
    """X uniform in [0, 1]^d, a smooth target plus noise, lengthscales around 0.3 sqrt(d)"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(4 * X[:, 0]) + (np.cos(3 * X[:, 1]) if d > 1 else 0.0) + 0.2 * rng.standard_normal(N)
    ls = rng.uniform(0.25, 0.4, d) * np.sqrt(d) if ell is None else np.full(d, float(ell))
    return X, y, np.concatenate([ls, [scale, noise, 0.7 if kind == "Periodic" else 1.0]])


def elbo_problem(kind, M, N, d, seed, noise=0.1, xu_is_x=False):
    """inducing points near a random subset of the training inputs (on it when xu_is_x)"""
    X, y, theta = mll_problem(kind, N, d, seed, noise)
    rng = np.random.default_rng(seed + 1)
    if xu_is_x:
        Xu = X.copy()
    else:
        Xu = X[rng.choice(N, M, replace=M > N)] + 0.02 * rng.standard_normal((M, d))
    return Xu, X, y, theta
