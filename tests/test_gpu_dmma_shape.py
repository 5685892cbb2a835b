"""The m16n8k4 DMMA kernels (gemm_tma_kernel, every gemm_nt_kernel configuration, trsm_strip_kernel) at the edges of
their fragment mapping: every k from 1 to 40 (one, two and three 16-wide k-slices, partly zero-filled), ragged m and n
of 16 q + r that cut an m16 tile after 1, 8, 9 and 15 rows, and the tail launch of the persistent kernel.  Errors are
measured against a DGEMM bound (k 2^-52 |a_i| |b_j| plus the rounding of the update of C); the TMA path and the
cp.async path must still agree bit for bit."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg as sla

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def check_update(C, C0, A, B, lower):
    """C == C0 - A B^T within a DGEMM bound (lower triangle only, the rest untouched, when `lower`)"""
    ref = C0 - A @ B.T
    k = A.shape[1]
    scale = np.linalg.norm(A, axis=1)[:, None] * np.linalg.norm(B, axis=1)[None, :] + np.abs(C0) + np.abs(ref)
    err = np.abs(C - ref) / scale
    if lower:
        mask = np.tril(np.ones(C.shape, bool))
        np.testing.assert_array_equal(C[~mask], C0[~mask])
        err = err[mask]
    assert err.max() <= max(k, 2) * 2.0 ** -52, err.max()


def counted(ctx, fn):
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


@pytest.mark.parametrize("lower", [False, True])
@pytest.mark.parametrize("k", list(range(1, 41)) + [8191])
def test_tma_path_every_k(ctx, k, lower):
    m = n = 2048
    rng = np.random.default_rng(k + 1000 * lower)
    A = rng.standard_normal((m, k))
    B = A if lower else rng.standard_normal((n, k))
    C0 = rng.standard_normal((m, n))
    Cg, c = counted(ctx, lambda: ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0, lower_only=lower))
    assert c["gemm_tma"] == 1 and c["oz_mma"] == 0, c
    check_update(Cg, C0, A, B, lower)
    with ctx.options(tma=0):
        C2, c = counted(ctx, lambda: ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0, lower_only=lower))
    assert c["gemm_tma"] == 0 and c["gemm_nt"] == 1, c
    np.testing.assert_array_equal(Cg, C2)


@pytest.mark.parametrize("r", [1, 8, 9, 15])
def test_tma_tail_ragged(ctx, r):
    """more 128x128 tiles than SMs and a partial last wave: the last tiles go to the 64x64 quarter-tile launch, whose
    tiles hold the ragged row and column edges"""
    sm = ctx.device_info()["sm_count"]
    tn = 12
    tm = sm // tn + 1                       # tm * tn > sm, not a multiple of it (tn = 12 < sm)
    assert tm * tn > sm and (tm * tn) % sm
    m, n, k = 128 * (tm - 1) + r, 128 * (tn - 1) + 16 + r, 37
    rng = np.random.default_rng(r)
    A, B, C0 = rng.standard_normal((m, k)), rng.standard_normal((n, k)), rng.standard_normal((m, n))
    Cg, c = counted(ctx, lambda: ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0))
    assert c["gemm_tma"] == 1 and c["gemm_nt"] == 1, c
    check_update(Cg, C0, A, B, False)
    with ctx.options(tma=0):
        C2 = ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0)
    np.testing.assert_array_equal(Cg, C2)


# b2gp_debug_gemm_cfg: 6 = 32x128 (1x8 warps), 7 = 64x128 (2x4), 8 = 64x64 (2x4, the lower-only and tail tile)
@pytest.mark.parametrize("cfg,lower", [(6, 0), (7, 0), (8, 0), (8, 1)])
@pytest.mark.parametrize("r", [1, 8, 9, 15])
def test_small_tile_configs_ragged(ctx, cfg, lower, r):
    m = 16 * 13 + r
    n = m if lower else 16 * 11 + r
    k = 16 * 3 + r
    rng = np.random.default_rng(cfg * 100 + r)
    A = rng.standard_normal((m, k))
    B = A if lower else rng.standard_normal((n, k))
    C0 = rng.standard_normal((m, n))
    dA, dB, dC = ctx.to_device(A), ctx.to_device(B), ctx.to_device(C0)
    fn = ctx.lib.b2gp_debug_gemm_cfg
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_int] + [C.c_int64] * 3 + [C.c_void_p, C.c_int64] * 3 + [C.c_int, C.POINTER(C.c_double)]
    ms = C.c_double()
    rc = fn(ctx.h, cfg, m, n, k, dA.ptr, k, dB.ptr, k, dC.ptr, n, lower, C.byref(ms))   # C = C0 - A B^T
    assert rc == 0, ctx.lib.b2gp_last_error(ctx.h)
    Cg = dC.download((m, n))
    for d in (dA, dB, dC):
        d.free()
    check_update(Cg, C0, A, B, bool(lower))


@pytest.mark.parametrize("n", [200, 256])
def test_trsm_strip_kernel(ctx, n):
    rng = np.random.default_rng(n)
    G = rng.standard_normal((n, n))
    A = G @ G.T / n + np.eye(n)
    B = rng.standard_normal((301, n))
    with ctx.options(ozaki=0):
        L, info = ctx.potrf(A)
        assert info == 0
        X, c = counted(ctx, lambda: ctx.trsm_lower(L, B))
    assert c["trsm_strip"] == 1 and c["gemm_nt"] == c["gemm_tma"] == 0, c
    ref = sla.solve_triangular(np.tril(L), B.T, lower=True).T
    np.testing.assert_allclose(X, ref, rtol=0, atol=1e-12 * np.abs(ref).max())


@pytest.mark.parametrize("shape", range(4))
def test_dmma_peak_probe(ctx, shape):
    fn = ctx.lib.b2gp_debug_dmma_peak
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    tf, ms = C.c_double(), C.c_double()
    rc = fn(ctx.h, shape, 4096, 1, C.byref(tf), C.byref(ms))
    assert rc == 0, ctx.lib.b2gp_last_error(ctx.h)
    assert np.isfinite(tf.value) and tf.value > 0 and ms.value > 0
