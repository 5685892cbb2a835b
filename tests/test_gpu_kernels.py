"""GPU: each CUDA kernel through the C-ABI against the oracle / NumPy on the same seeded inputs."""
import numpy as np
import pytest
import scipy.linalg as sla

import oracle
from conftest import assert_close

pytestmark = pytest.mark.gpu

KMAP = {"RBF": oracle.rbf_kernel, "Matern": oracle.matern_kernel, "Periodic": oracle.periodic_kernel}


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def spd(rng, n, cond=1e3):
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    ev = np.geomspace(1.0, cond, n)
    A = (Q * ev) @ Q.T
    return (A + A.T) / 2


# ------------------------------------------------------------------ Gram
def test_gram_golden(ctx, golden):
    """against the vectors produced by the reference's own kernel functions; bar: rtol 1e-13 (SURVEY 8c)"""
    for tag in (str(c) for c in golden["gram_cases"]):
        kname = tag.split("_")[1]
        X, Z, ell = golden[tag + "_X"], golden[tag + "_Z"], golden[tag + "_ell"]
        K = ctx.gram(kname, X, Z, ell, 1.3, 0.9, diag_add=0.05 + 1e-6)
        np.testing.assert_allclose(K, golden[tag + "_K"], rtol=1e-13, atol=1e-14, err_msg=tag)
    X = golden["gramself_X"]
    for kname in KMAP:
        K = ctx.gram(kname, X, X, [0.4, 0.6], 2.0, 1.0, diag_add=0.1 + 1e-6)
        np.testing.assert_allclose(K, golden[f"gramself_{kname}_K"], rtol=1e-13, atol=1e-14)


@pytest.mark.parametrize("kname", ["RBF", "Matern", "Periodic"])
@pytest.mark.parametrize("n,m,d", [(1, 1, 1), (63, 129, 2), (64, 128, 3), (257, 31, 5), (300, 300, 1), (1000, 777, 3)])
def test_gram_vs_oracle(ctx, kname, n, m, d):
    rng = np.random.default_rng(n * 1000 + m + d)
    X, Z = rng.uniform(-2, 2, (n, d)), rng.uniform(-2, 2, (m, d))
    ell = rng.uniform(0.3, 2.0, d)
    params = {"k_length": ell, "k_scale": 0.7, "period": 1.7}
    ref = KMAP[kname](X, Z, params, 0.2, jitter=1e-6)
    K = ctx.gram(kname, X, Z, ell, 0.7, 1.7, diag_add=0.2 + 1e-6)
    np.testing.assert_allclose(K, ref, rtol=1e-13, atol=1e-14)


def test_gram_lower_only_and_diag(ctx):
    rng = np.random.default_rng(5)
    X = rng.uniform(0, 1, (333, 2))
    params = {"k_length": np.array([0.3, 0.5]), "k_scale": 1.1}
    ref = oracle.matern_kernel(X, X, params, 0.1, jitter=1e-6)
    K = ctx.gram("Matern", X, X, [0.3, 0.5], 1.1, diag_add=0.1 + 1e-6, lower_only=True)
    np.testing.assert_allclose(np.tril(K), np.tril(ref), rtol=1e-13, atol=1e-14)
    assert np.all(np.triu(K, 1) == 0)
    # k(x,x) = k_scale (+ noise + jitter): SURVEY 8c closed form
    Kr = ctx.gram("RBF", X, X, [0.3, 0.5], 1.1, diag_add=0.25)
    np.testing.assert_allclose(np.diag(Kr), 1.1 + 0.25, rtol=1e-15)
    # symmetric
    np.testing.assert_allclose(Kr, Kr.T, rtol=0, atol=1e-15)


def test_gram_no_diag_when_shapes_differ(ctx):
    X = np.linspace(0, 1, 10)[:, None]
    K = ctx.gram("RBF", X, X[:7], [0.5], 1.0, diag_add=5.0)
    assert K.shape == (10, 7) and K.max() <= 1.0 + 1e-15


# ------------------------------------------------------------------ GEMM / SYRK (DMMA)
@pytest.mark.parametrize("m,n,k", [(1, 1, 1), (8, 8, 4), (128, 128, 16), (130, 70, 33), (257, 129, 300), (64, 512, 1000)])
def test_gemm_nt(ctx, m, n, k):
    rng = np.random.default_rng(m + n + k)
    A, B, C0 = rng.standard_normal((m, k)), rng.standard_normal((n, k)), rng.standard_normal((m, n))
    C = ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0)
    ref = C0 - A @ B.T
    np.testing.assert_allclose(C, ref, rtol=0, atol=1e-13 * max(1.0, k ** 0.5) * np.abs(ref).max())
    C = ctx.gemm_nt(A, B, np.full((m, n), np.nan), alpha=2.0, beta=0.0)       # beta = 0 must not read C
    np.testing.assert_allclose(C, 2 * A @ B.T, rtol=0, atol=1e-13 * max(1.0, k ** 0.5) * np.abs(ref).max())


@pytest.mark.parametrize("n,k", [(5, 3), (128, 128), (300, 64), (513, 257)])
def test_syrk_lower(ctx, n, k):
    rng = np.random.default_rng(n + k)
    A, C0 = rng.standard_normal((n, k)), rng.standard_normal((n, n))
    C = ctx.gemm_nt(A, A, C0, alpha=-1.0, beta=1.0, lower_only=True)
    ref = C0 - A @ A.T
    np.testing.assert_allclose(np.tril(C), np.tril(ref), rtol=0, atol=1e-13 * k ** 0.5 * np.abs(ref).max())
    np.testing.assert_array_equal(np.triu(C, 1), np.triu(C0, 1))               # strict upper untouched


@pytest.mark.parametrize("m,n,k,lower", [(2048, 2048, 300, False), (1700, 2333, 77, False), (2100, 2100, 257, True),
                                           (4096, 4096, 1024, True)])
def test_gemm_large_tma_path(ctx, m, n, k, lower):
    """>= 112 tiles of 128x128: the persistent TMA / mbarrier kernel (gemm_tma.cuh), ragged edges zero-filled by TMA;
    and the same call with the TMA path switched off must give the same bits (same DMMA accumulation order)"""
    rng = np.random.default_rng(m + k)
    A = rng.standard_normal((m, k))
    B = A if lower else rng.standard_normal((n, k))
    C0 = rng.standard_normal((m, n))
    C = ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0, lower_only=lower)
    ref = C0 - A @ B.T
    tol = 1e-13 * k ** 0.5 * np.abs(ref).max()
    if lower:
        np.testing.assert_allclose(np.tril(C), np.tril(ref), rtol=0, atol=tol)
        np.testing.assert_array_equal(np.triu(C, 1), np.triu(C0, 1))
    else:
        np.testing.assert_allclose(C, ref, rtol=0, atol=tol)
    with ctx.options(tma=0):
        C2 = ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0, lower_only=lower)
    np.testing.assert_array_equal(C, C2)


@pytest.mark.parametrize("m,n,k,lower", [(2500, 1300, 700, False), (3000, 3000, 1536, True), (1025, 8192, 4096, False)])
def test_int8_wgmma_gemm(ctx, m, n, k, lower):
    """the rank-k update through the int8 digit-plane kernel (ozaki.cuh): rows of very different magnitude (each row
    carries its own power-of-two scale), ragged m / n / k; error measured against |a_i| |b_j| like a DGEMM's"""
    rng = np.random.default_rng(m + n + k)
    A = rng.standard_normal((m, k)) * np.exp(rng.normal(0, 3, (m, 1)))
    B = A if lower else rng.standard_normal((n, k)) * np.exp(rng.normal(0, 3, (n, 1)))
    C0 = rng.standard_normal((m, n))
    ref = C0 - A @ B.T
    # a DGEMM-style bound: rounding of the product (|a_i| |b_j|) plus rounding of the update of C itself
    scale = np.linalg.norm(A, axis=1)[:, None] * np.linalg.norm(B, axis=1)[None, :] + np.abs(C0) + np.abs(ref)
    errs = {}
    for planes in (0, 7, 6):
        with ctx.options(ozaki=planes):
            before = ctx.path_counts()["oz_mma"]
            C = ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0, lower_only=lower)
            assert ctx.path_counts()["oz_mma"] - before == (1 if planes else 0)   # the kernel the error bar is for
        mask = np.tril(np.ones((m, n), bool)) if lower else np.ones((m, n), bool)
        errs[planes] = (np.abs(C - ref) / scale)[mask].max()
        if lower:
            np.testing.assert_array_equal(C[~mask], C0[~mask])
    assert errs[0] <= 3e-15 and errs[7] <= 2e-14 and errs[6] <= 5e-13, errs
    # alpha, and a B different from A with lower_only off
    with ctx.options(ozaki=7):
        C = ctx.gemm_nt(A, B, C0, alpha=0.5, beta=1.0, lower_only=lower)
    ref2 = C0 + 0.5 * A @ B.T
    scale2 = scale + np.abs(ref2)
    assert (np.abs(C - ref2) / scale2)[np.tril(np.ones((m, n), bool)) if lower else np.ones((m, n), bool)].max() <= 2e-14


# ------------------------------------------------------------------ Cholesky + triangular solve
@pytest.mark.parametrize("n", [1, 2, 31, 64, 65, 127, 128, 129, 200, 256, 300, 511, 777, 1024, 1500, 4100])
def test_potrf(ctx, n):
    rng = np.random.default_rng(n)
    A = spd(rng, n)
    L, info = ctx.potrf(A)
    assert info == 0
    Lt = np.tril(L)
    # reconstruction bound of SURVEY 8c: |L L^T - K|_F / |K|_F <= 1e-14 sqrt(N)
    assert np.linalg.norm(Lt @ Lt.T - A) / np.linalg.norm(A) <= 1e-14 * max(1.0, n ** 0.5)
    ref = sla.cholesky(A, lower=True)
    np.testing.assert_allclose(Lt, ref, rtol=0, atol=1e-10 * np.abs(ref).max())
    np.testing.assert_array_equal(np.triu(L, 1), np.triu(A, 1))                # strict upper untouched


@pytest.mark.parametrize("n,nrhs", [(129, 5), (256, 32), (300, 77), (511, 31), (512, 1025), (1000, 64), (2048, 300)])
def test_trsm_strip_kernel_matches_recursion(ctx, n, nrhs):
    """the one-launch strip solve (factors up to 512 wide, potrf.cuh) against the recursive GEMM formulation it replaces"""
    rng = np.random.default_rng(7 * n + nrhs)
    A = spd(rng, n)
    B = rng.standard_normal((nrhs, n))
    out = {}
    assert ctx.get_option("ozaki") == 0          # with the int8 path on, >= 1024 rows would take the panel route, not the strip kernel
    for strip in (0, 256, 512):
        with ctx.options(trsm_strip=strip):
            L, info = ctx.potrf(A)
            assert info == 0
            before = ctx.path_counts()
            out[strip] = (np.tril(L), ctx.trsm_lower(L, B))
            after = ctx.path_counts()
            assert (after["trsm_strip"] > before["trsm_strip"]) == (strip > 0) and after["panel_solve"] == before["panel_solve"]
    ref = sla.solve_triangular(out[0][0], B.T, lower=True).T
    for strip in (256, 512):
        np.testing.assert_allclose(out[strip][0], out[0][0], rtol=0, atol=1e-12 * np.abs(out[0][0]).max())
        np.testing.assert_allclose(out[strip][1], ref, rtol=0, atol=1e-11 * np.abs(ref).max())


def test_potrf_not_positive_definite(ctx):
    rng = np.random.default_rng(0)
    A = spd(rng, 200)
    A[150, 150] = -1.0
    L, info = ctx.potrf(A)
    assert info == 151
    A = spd(rng, 40)
    A[0, 0] = 0.0
    assert ctx.potrf(A)[1] == 1


@pytest.mark.parametrize("n,nrhs", [(1, 1), (100, 3), (128, 128), (300, 17), (640, 200), (1000, 1), (512, 33), (1536, 1025)])
def test_trsm(ctx, n, nrhs):
    rng = np.random.default_rng(n + nrhs)
    A = spd(rng, n)
    L, info = ctx.potrf(A)
    assert info == 0
    B = rng.standard_normal((nrhs, n))
    X = ctx.trsm_lower(L, B)
    ref = sla.solve_triangular(np.tril(L), B.T, lower=True).T
    np.testing.assert_allclose(X, ref, rtol=0, atol=1e-11 * np.abs(ref).max())
