"""Test-only stand-in for gpax_b200.distributed.GpuOps: the same local-compute interface on CPU torch
tensors with NumPy/SciPy + the oracle's kernel functions.  It exists so that the HOST LOGIC of the
multi-rank algorithms (ownership, panel broadcast, fan-in reduce, all-reduce) runs under gloo with
world_size 2 on a machine without GPUs.  It is never importable from the product package.
tests/test_gpu_dist_single.py runs both on identical inputs and requires the same results, info codes included."""
import numpy as np
import scipy.linalg as sla
import torch

import oracle

KMAP = {"RBF": oracle.rbf_kernel, "Matern": oracle.matern_kernel, "Periodic": oracle.periodic_kernel}
LEAF = 128      # the inverted diagonal blocks b2gp_potrf_inv exports are LEAF x LEAF


def params_of(theta, d):
    return {"k_length": np.asarray(theta[:d]), "k_scale": float(theta[d]), "noise": float(theta[d + 1]),
            "period": float(theta[d + 2])}


def chol(a):
    """(L, info) of the lower triangle of a: info = 0, or the 1-based index of the first non-positive pivot, as the
    library's factorisations report it (LAPACK potrf's convention)"""
    full = np.tril(a) + np.tril(a, -1).T
    L, info = sla.lapack.dpotrf(full, lower=1, clean=1)
    if info == 0:     # a NaN pivot fails too (the library tests !(pivot > 0)); not every LAPACK build checks for it
        bad = np.flatnonzero(~(np.diag(L) > 0.0))
        info = int(bad[0]) + 1 if bad.size else 0
    return np.tril(L), int(info)


class NumpyOps:
    def empty(self, shape):
        return torch.zeros(shape, dtype=torch.float64)

    zeros = empty

    def from_numpy(self, a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))

    def to_numpy(self, t):
        return t.numpy().copy()

    def sync(self):
        pass

    def gram(self, kind, X, Z, theta, diag_add, same, out):
        d = X.shape[1]
        Xn, Zn = X.numpy(), Z.numpy()
        K = KMAP[kind](Xn, Zn, params_of(theta, d), 0.0, jitter=0.0)
        if Xn.shape == Zn.shape:      # the oracle applied (0 + 0) * I
            pass
        if same:
            n = min(K.shape)
            K = K.copy()
            K[np.arange(n), np.arange(n)] += diag_add
        out.numpy()[...] = K

    def potrf_inv(self, A, linv):
        """lower triangle of A <- L; linv <- inv(L_bb) of every LEAF-wide diagonal block, row-major LEAF x LEAF, zero above
        the diagonal and outside a ragged last block; returns info (A's contents are NaN when info != 0)"""
        a = A.numpy()
        n = a.shape[0]
        L, info = chol(a)
        if info:
            a[...] = np.nan
            return info
        a[np.tril_indices(n)] = L[np.tril_indices(n)]
        blocks = linv.numpy().reshape(-1, LEAF, LEAF)
        blocks[...] = 0.0
        for b in range(-(-n // LEAF)):
            lo, hi = b * LEAF, min(n, (b + 1) * LEAF)
            blocks[b, :hi - lo, :hi - lo] = sla.solve_triangular(L[lo:hi, lo:hi], np.eye(hi - lo), lower=True)
        return 0

    def trsm_inv(self, L, linv, B):
        if B.shape[0] == 0:
            return
        b = B.numpy()
        b[...] = sla.solve_triangular(np.tril(L.numpy()), b.T, lower=True, check_finite=False).T

    def gemm_nt(self, A, B, C, alpha, beta, lower=False):
        c = C.numpy()
        prod = alpha * (A.numpy() @ B.numpy().T)
        c[...] = prod if beta == 0.0 else beta * c + prod

    def rowdot(self, R, w, dot, nrm, accumulate):
        r = R.numpy()
        if dot is not None:
            v = r @ w.numpy()
            dot.numpy()[...] = dot.numpy() + v if accumulate else v
        if nrm is not None:
            v = (r * r).sum(1)
            nrm.numpy()[...] = nrm.numpy() + v if accumulate else v

    def copy(self, dst, src):
        dst.numpy()[...] = src.numpy()

    def sparse_partial(self, kind, Xu, Xtr, y, theta, jitter, Kpart, cpart):
        """info: the first bad pivot of chol(Kuu + jitter I) (Kpart / cpart NaN then)"""
        d = Xu.shape[1]
        p = params_of(theta, d)
        Kuu = KMAP[kind](Xu.numpy(), Xu.numpy(), p, 0.0, jitter=jitter)
        Luu, info = chol(Kuu)
        if info:
            Kpart.numpy()[...] = np.nan
            cpart.numpy()[...] = np.nan
            return info
        W = sla.solve_triangular(Luu, KMAP[kind](Xu.numpy(), Xtr.numpy(), p, 0.0, jitter=0.0), lower=True)
        Kpart.numpy()[...] = np.tril(W @ W.T / p["noise"])
        cpart.numpy()[...] = W @ y.numpy() / p["noise"]
        return 0

    def sparse_finish(self, kind, Xu, Ksum, csum, Xnew, theta, noiseless, jitter, mean, var, cov):
        """info: > 0 the first bad pivot of chol(Kuu + jitter I), < 0 minus the first bad pivot of chol(Ksum + I);
        every output NaN then"""
        d = Xu.shape[1]
        p = params_of(theta, d)
        k = KMAP[kind]
        Kuu = k(Xu.numpy(), Xu.numpy(), p, 0.0, jitter=jitter)
        Luu, info_u = chol(Kuu)
        Kl = np.tril(Ksum.numpy())
        L, info_k = chol(Kl + np.eye(Kl.shape[0]))
        info = info_u if info_u else -info_k
        if info:
            for out in (mean, var, cov):
                if out is not None:
                    out.numpy()[...] = np.nan
            return info
        Ws = sla.solve_triangular(Luu, k(Xu.numpy(), Xnew.numpy(), p, 0.0, jitter=0.0), lower=True)
        Lc = sla.solve_triangular(L, csum.numpy(), lower=True)
        LWs = sla.solve_triangular(L, Ws, lower=True)
        mean.numpy()[...] = Lc @ LWs
        noise_p = p["noise"] * (0.0 if noiseless else 1.0)
        Kss = k(Xnew.numpy(), Xnew.numpy(), p, noise_p, jitter=jitter)
        c = Kss - Ws.T @ Ws + LWs.T @ LWs
        if var is not None:
            var.numpy()[...] = np.diag(c)
        if cov is not None:
            cov.numpy()[...] = c
        return 0
