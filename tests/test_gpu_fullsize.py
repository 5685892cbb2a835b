"""GPU: BASELINE.json's full sizes through size-independent properties (the oracle needs minutes there)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import gpax_b200
    return gpax_b200.default_context()


def test_factor_reconstructs_K_at_N16384(ctx):
    """|L L^T - K|_F / |K|_F <= 1e-14 sqrt(N) (SURVEY 8c) at the headline size, all on the device:
    K is rebuilt by the Gram kernel, L L^T by the SYRK kernel, the difference measured through row reductions."""
    from gpax_b200 import _ffi
    N, d = 16384, 3
    rng = np.random.default_rng(4)
    X = ctx.to_device(rng.uniform(0, 1, (N, d)))
    ell = np.full(d, 0.3)
    K, L = ctx.alloc((N, N)), ctx.alloc((N, N))
    fl = _ffi.FLAG_DEVICE_PTRS
    for buf in (K, L):
        ctx._check(ctx.lib.b2gp_gram(ctx.h, 0, X.ptr, N, X.ptr, N, d, _ffi._ptr(ell), 1.0, 1.0, 0.1 + 1e-6, 1, buf.ptr, N, fl))
    info = C.c_int(0)
    ctx._check(ctx.lib.b2gp_potrf(ctx.h, N, L.ptr, N, C.byref(info), fl))
    assert info.value == 0
    # The leading n x n block of L is exactly the factor of the leading block of K: check the reconstruction bound
    # there (downloading 2 GiB row by row would dominate the test), then a last-row identity that depends on all
    # 16384 columns.
    n = 4096
    Lb = np.tril(np.ascontiguousarray(_download_block(ctx, L, N, n)))
    Kb = _download_block(ctx, K, N, n)
    Kb = np.tril(Kb) + np.tril(Kb, -1).T
    rec = ctx.gemm_nt(Lb, Lb, lower_only=False)
    assert np.linalg.norm(rec - Kb) / np.linalg.norm(Kb) <= 1e-14 * np.sqrt(N)
    # and the last diagonal entries (which depend on every earlier column) against an independent identity:
    # sum_j L_ij^2 == K_ii for the last row
    row = _download_rows(ctx, L, N, N - 1, 1)[0]
    assert abs(np.dot(row, row) - (1.0 + 0.1 + 1e-6)) <= 1e-12
    for b in (X, K, L):
        b.free()


def _download_block(ctx, dev, ld, n):
    full = np.empty((n, n))
    tmp = np.empty(ld)
    for i in range(n):       # row by row (n small): uses the plain d2h entry point
        ctx._check(ctx.lib.b2gp_d2h(ctx.h, C.c_void_p(tmp.ctypes.data), C.c_void_p(dev.ptr.value + i * ld * 8), n * 8))
        full[i] = tmp[:n]
    return full


def _download_rows(ctx, dev, ld, r0, nrows):
    out = np.empty((nrows, ld))
    ctx._check(ctx.lib.b2gp_d2h(ctx.h, C.c_void_p(out.ctypes.data), C.c_void_p(dev.ptr.value + r0 * ld * 8), nrows * ld * 8))
    return out


def test_posterior_interpolates_at_N16384(ctx):
    """with tiny noise the posterior mean at training points reproduces y and the variance collapses (closed form of
    SURVEY 8c), N=16384 d=3; plus draw-order independence: the same theta twice in a batch gives identical bits"""
    N, d, P = 16384, 3, 256
    rng = np.random.default_rng(4)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(3 * X[:, 0]) * np.cos(2 * X[:, 1]) + X[:, 2]
    theta = np.array([[0.3, 0.3, 0.3, 1.0, 1e-4, 1.0]] * 2)          # cond(K) ~ 1e4 / 1e-4
    out = ctx.posterior("Matern", X, y, X[:P], theta, noiseless=True, want=("mean", "var"))
    assert (out["info"] == 0).all()
    assert np.abs(out["mean"][0] - y[:P]).max() < 5e-3
    assert (out["var"][0] > 0).all() and out["var"][0].max() < 2e-4
    np.testing.assert_array_equal(out["mean"][0], out["mean"][1])
    np.testing.assert_array_equal(out["var"][0], out["var"][1])


def test_many_draws_stream_through_few_workspaces(ctx):
    """S = 24 draws at N = 4096 (the reference would hold 24 x 128 MiB at once): linearity in y as the property:
    posterior mean is linear in the targets, mean(y1 + 2 y2) == mean(y1) + 2 mean(y2) to rounding"""
    N, d, P, S = 4096, 2, 128, 24
    rng = np.random.default_rng(9)
    X, Xn = rng.uniform(0, 1, (N, d)), rng.uniform(0, 1, (P, d))
    y1, y2 = rng.standard_normal(N), rng.standard_normal(N)
    theta = np.column_stack([np.exp(rng.normal(np.log(0.3), 0.1, (S, d))), np.exp(rng.normal(0, 0.1, S)),
                             np.exp(rng.normal(np.log(0.1), 0.1, S)), np.ones(S)])
    with ctx.options(streams=4):
        a = ctx.posterior("RBF", X, y1, Xn, theta, want=("mean",))["mean"]
        b = ctx.posterior("RBF", X, y2, Xn, theta, want=("mean",))["mean"]
        c = ctx.posterior("RBF", X, y1 + 2 * y2, Xn, theta, want=("mean",))["mean"]
    scale = np.abs(c).max()
    np.testing.assert_allclose(c, a + 2 * b, rtol=0, atol=1e-9 * scale)


def test_int8_wgmma_path_matches_fp64_dmma_path(ctx):
    """N = 8192 (large enough for the int8 digit-plane kernel to take the trailing updates): the posterior through the
    int8 path with 7 base-256 planes agrees with the all-fp64 DMMA path to the parity bar (1e-9, scale-relative) at
    cond(K) ~ 1e5, and so does 6 planes to 1e-7; the factor itself agrees to 1e-12 of its scale.  (The comparison
    with the oracle at this size and at N = 16384 is tests/test_gpu_baseline_sizes.py.)"""
    import ctypes as C
    from gpax_b200 import _ffi
    N, d, P = 8192, 2, 200
    rng = np.random.default_rng(21)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(4 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.05 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    theta = np.array([[0.25, 0.3, 1.0, 1e-3, 1.0]])       # noise 1e-3 -> cond(K) ~ N * scale / noise ~ 1e5 .. 1e6 effective
    res = {}
    for planes in (0, 7, 6):
        with ctx.options(ozaki=planes):
            ctx.set_option("drop_factor_cache", 1)
            before = ctx.path_counts()
            res[planes] = ctx.posterior("Matern", X, y, Xn, theta, want=("mean", "var"))
            moved = {k: v - before[k] for k, v in ctx.path_counts().items()}
        assert res[planes]["info"][0] == 0
        assert (moved["oz_mma"] > 0) == (moved["potrf_tall"] == 1) == (planes != 0), (planes, moved)
    ref = res[0]
    for planes, tol in ((7, 1e-9), (6, 1e-7)):
        for k in ("mean", "var"):
            err = np.abs(res[planes][k] - ref[k]).max() / np.abs(ref[k]).max()
            print(f"planes={planes} {k}: max scaled deviation from the fp64 DMMA path {err:.2e}")
            assert err <= tol, (planes, k, err)
    # factor level: L from both paths on a device-resident K
    dX = ctx.to_device(X)
    ell = np.array([0.25, 0.3])
    Ls = {}
    for planes in (0, 7):
        K = ctx.alloc((N, N))
        ctx._check(ctx.lib.b2gp_gram(ctx.h, 1, dX.ptr, N, dX.ptr, N, d, _ffi._ptr(ell), 1.0, 1.0, 1e-3 + 1e-6, 1, K.ptr, N,
                                     _ffi.FLAG_DEVICE_PTRS))
        info = C.c_int(0)
        with ctx.options(ozaki=planes):
            ctx._check(ctx.lib.b2gp_potrf(ctx.h, N, K.ptr, N, C.byref(info), _ffi.FLAG_DEVICE_PTRS))
        assert info.value == 0
        Ls[planes] = _download_rows(ctx, K, N, N - 64, 64)      # the last 64 rows depend on every update
        K.free()
    mask = np.tril(np.ones((N, N), bool))[N - 64:]
    dev = np.abs(Ls[7] - Ls[0])[mask].max() / np.abs(Ls[0][mask]).max()
    print(f"factor rows {N-64}..{N}: max scaled deviation {dev:.2e}")
    assert dev <= 1e-12
    dX.free()
