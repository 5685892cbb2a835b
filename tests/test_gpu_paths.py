"""GPU: every solver path under options that are NAMED in the test, with a witness of which kernels ran.

The library picks its kernels from context options (`ozaki`, `panel`, `tall_min`, `trsm_strip`, `oz_min_tiles`, ...) and
from sizes.  A numeric test alone cannot tell a dispatch regression from a correct run -- every path computes the same
posterior -- so each test here sets its options on a context of its own, reads the cumulative path counters
(`Context.path_counts()`, b2gp_debug_path_counts) around the call and asserts both the numbers and the route.  Nothing in
this file touches `gpax_b200.default_context()`, so the verdicts do not depend on what ran before."""
import functools
import os

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse.linalg as spla

import oracle
from conftest import assert_close
from oracle import ozaki_oracle as oz

pytestmark = pytest.mark.gpu

RTOL = 1e-9   # the parity bar, at cond(K) <= 1e5; scaled by cond / 1e5 beyond (as in test_gpu_posterior.py)


@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def counted(ctx, fn):
    """fn() and the path counters it moved"""
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


def theta_of(params, d):
    ell = np.broadcast_to(np.asarray(params["k_length"], dtype=float).reshape(-1), (d,))
    return np.concatenate([ell, [params["k_scale"], params["noise"], params.get("period", 1.0)]])


def spd(rng, n, cond=1e3):
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    ev = np.geomspace(1.0, cond, n)
    A = (Q * ev) @ Q.T
    return (A + A.T) / 2


PARAMS = {"k_length": np.array([0.25, 0.35]), "k_scale": 1.1, "noise": 0.05, "period": 0.9}
KERNEL_AT = {2047: "Matern", 2048: "Periodic", 2500: "RBF", 3100: "Matern"}


@functools.lru_cache(maxsize=2)
def problem(kname, N, P):
    """seeded inputs, the Cholesky oracle's posterior and the tolerance at this conditioning (lambda_max by Lanczos,
    lambda_min >= noise + jitter)"""
    rng = np.random.default_rng(N + P)
    d = 2
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    rmean, rcov = oracle.exact_posterior_chol(X, y, Xn, PARAMS, kname)
    K = oracle.get_kernel(kname)(X, X, PARAMS, PARAMS["noise"])
    cond = float(spla.eigsh(K, k=1, which="LA", return_eigenvectors=False, tol=1e-4)[0]) / (PARAMS["noise"] + 1e-6)
    return X, y, Xn, rmean, rcov, RTOL * max(1.0, cond / 1e5), cond


def check_posterior(out, rmean, rcov, tol, what):
    assert out["info"][0] == 0, what
    assert_close(out["mean"][0], rmean, tol, "mean " + what)
    assert_close(out["var"][0], np.diag(rcov), tol, "var " + what)
    assert_close(out["cov"][0], rcov, tol, "cov " + what)


# ------------------------------------------------------------------ 1. options
DEFAULTS = {"ozaki": 0, "streams": 2, "panel": 1024, "tall_min": 2048, "trsm_strip": 256, "oz_cluster": 2, "tma": 1,
            "enqueue_threads": 1, "big_grid": 0, "oz_debug": 0}
OTHER = {"ozaki": 7, "streams": 5, "panel": 256, "tall_min": 4096, "trsm_strip": 512, "oz_cluster": 1, "tma": 0,
         "enqueue_threads": 0, "big_grid": 100, "oz_debug": 1, "oz_min_tiles": 17}


def test_fresh_context_reports_the_documented_defaults_and_every_option_reads_back(ctx):
    from gpax_b200._ffi import B200GPError
    sm = ctx.device_info()["sm_count"]
    got = {k: ctx.get_option(k) for k in OTHER}
    assert got == dict(DEFAULTS, oz_min_tiles=sm)
    for k, v in OTHER.items():
        ctx.set_option(k, v)
        assert ctx.get_option(k) == v, k
        assert {q: ctx.get_option(q) for q in OTHER if q != k} == {q: w for q, w in got.items() if q != k}, f"{k} moved another option"
        ctx.set_option(k, got[k])
    for v in (-1, 6):
        ctx.set_option("ozaki", v)
        assert ctx.get_option("ozaki") == v
    ctx.set_option("ozaki", 0)
    with ctx.options(ozaki=-1, panel=512):
        assert (ctx.get_option("ozaki"), ctx.get_option("panel")) == (-1, 512)
    with pytest.raises(ZeroDivisionError):
        with ctx.options(streams=7):
            1 / 0
    assert {k: ctx.get_option(k) for k in OTHER} == got                # restored, also when the block raises
    for bad in ("drop_factor_cache", "no_such_option"):                # an action and an unknown key hold no value
        with pytest.raises(B200GPError):
            ctx.get_option(bad)
    with pytest.raises(B200GPError):
        ctx.set_option("ozaki", 5)
    assert ctx.get_option("ozaki") == 0


# ------------------------------------------------------------------ 2. posterior path matrix
@pytest.mark.parametrize("ozaki", [0, 7, 6, -1])
@pytest.mark.parametrize("N", [2047, 2048, 2500, 3100])
def test_posterior_paths_vs_oracle_with_witness(ctx, N, ozaki):
    """mean, var and the full covariance against the Cholesky oracle on either side of `tall_min`, under each `ozaki`
    value, and the route each combination must take"""
    P = 300          # P + 1 < 1024 rows: trsm_rec does not take the panel route on its own
    kname = KERNEL_AT[N]
    X, y, Xn, rmean, rcov, tol, cond = problem(kname, N, P)
    assert ctx.get_option("tall_min") == 2048 and ctx.get_option("panel") == 1024
    ctx.set_option("ozaki", ozaki)
    out, c = counted(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta_of(PARAMS, 2)[None], want=("mean", "var", "cov")))
    check_posterior(out, rmean, rcov, tol, f"{kname} N={N} ozaki={ozaki} cond(K) <= {cond:.1e}")
    assert c["potrf_diag"] == -(-N // 128) and c["gemm_nt"] + c["gemm_tma"] > 0, c
    if ozaki == 0:
        assert c["oz_mma"] == c["oz_slice"] == c["panel_solve"] == c["potrf_tall"] == c["trsm_tall"] == 0, c
    elif N >= 2048:
        assert c["potrf_tall"] == 1 and c["panel_solve"] == -(-N // 1024) and c["oz_mma"] >= c["panel_solve"], c
        assert c["oz_slice"] >= c["oz_mma"], c
    else:
        assert c["potrf_tall"] == c["panel_solve"] == c["trsm_tall"] == 0, c


def test_panel_width_changes_the_number_of_panel_solves(ctx):
    """one panel solve per diagonal block of the tall-panel factorisation; panel = 0 is the recursive fp64 scheme"""
    N, P, kname = 2500, 300, "RBF"
    X, y, Xn, rmean, rcov, tol, cond = problem(kname, N, P)
    theta = theta_of(PARAMS, 2)[None]
    ctx.set_option("ozaki", 7)
    means = {}
    for panel in (1024, 512, 256, 0):
        ctx.set_option("panel", panel)
        out, c = counted(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta, want=("mean", "var", "cov")))
        check_posterior(out, rmean, rcov, tol, f"panel={panel} cond(K) <= {cond:.1e}")
        want = -(-N // panel) if panel else 0
        assert c["panel_solve"] == want and c["potrf_tall"] == (1 if panel else 0), (panel, c)
        assert ctx.cache_hits() == 0                                    # setting `panel` drops the cached factor
        means[panel] = out["mean"][0]
    assert not np.array_equal(means[1024], means[0])                    # different arithmetic, same posterior
    # a failed factorisation gives NaN + info on this path too, not an exception
    ctx.set_option("panel", 1024)
    bad = ctx.posterior(kname, X, y, Xn, theta_of(dict(PARAMS, k_scale=-1.0), 2)[None], want=("mean", "cov"))
    assert bad["info"][0] > 0 and np.isnan(bad["mean"]).all() and np.isnan(bad["cov"]).all()


@pytest.mark.parametrize("streams", [1, 2, 3])
def test_default_path_batched_draws_and_samples(ctx, streams):
    """the shipped default (ozaki = 0) at N >= tall_min with S = 3 draws over 1, 2 (draws queued from one host thread per
    slot) and 3 streams: every draw against the oracle, samples from a fixed eps, equal theta -> identical bits"""
    N, P, d, S, n = 2048, 200, 2, 3, 2
    rng = np.random.default_rng(11)
    X, Xn = rng.uniform(0, 1, (N, d)), rng.uniform(0, 1, (P, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    samples = {"k_length": np.array([[0.3, 0.4], [0.25, 0.35], [0.3, 0.4]]), "k_scale": np.array([1.0, 1.2, 1.0]),
               "noise": np.array([0.1, 0.08, 0.1])}
    eps = rng.standard_normal((n, P))
    eps = np.broadcast_to(eps, (S, n, P)).copy()
    means, ysamp = [], []
    for s in range(S):
        m, cv = oracle.exact_posterior_chol(X, y, Xn, {k: v[s] for k, v in samples.items()}, "Matern")
        means.append(m)
        ysamp.append(m[None, :] + eps[s] @ np.linalg.cholesky(cv).T)       # y = mean + chol(cov) eps
    means, ysamp = np.stack(means), np.stack(ysamp)
    theta = np.concatenate([samples["k_length"], samples["k_scale"][:, None], samples["noise"][:, None], np.ones((S, 1))], 1)
    assert ctx.get_option("ozaki") == 0
    ctx.set_option("streams", streams)
    out, c = counted(ctx, lambda: ctx.posterior("Matern", X, y, Xn, theta, want=("mean", "var", "cov"), eps=eps))
    assert (out["info"] == 0).all()
    assert_close(out["mean"], means, RTOL, f"means, streams={streams}")
    assert_close(out["y_sampled"], ysamp, 1e-6, f"samples, streams={streams}")       # chol(cov) amplifies cov's rounding
    for k in ("mean", "var", "cov", "y_sampled"):
        np.testing.assert_array_equal(out[k][0], out[k][2], err_msg=f"{k}: draws 0 and 2 share theta, streams={streams}")
    assert c["oz_mma"] == c["oz_slice"] == c["panel_solve"] == c["potrf_tall"] == 0, c
    assert c["potrf_diag"] == S * (N // 128 + -(-P // 128)), c          # k_XX and the sampled covariance, per draw


# ------------------------------------------------------------------ 3. factor cache under each option set and across a toggle
@pytest.mark.parametrize("seq", ["all_fp64", "all_int8", "int8_then_fp64", "fp64_then_int8"])
def test_factor_cache_reuse_under_options(ctx, seq):
    """N = 2500, the first call factors and the later ones reuse the factor: at ozaki = 7 through the kept inverses of the
    diagonal blocks (trsm_tall), at ozaki = 0 through the recursion; when the option changes between the calls the reuse
    must fit the factor that is actually cached"""
    N, d = 2500, 2
    first, later = {"all_fp64": (0, 0), "all_int8": (7, 7), "int8_then_fp64": (7, 0), "fp64_then_int8": (0, 7)}[seq]
    rng = np.random.default_rng(N)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    params = {"k_length": np.array([0.3, 0.4]), "k_scale": 1.2, "noise": 0.05}
    K = oracle.matern_kernel(X, X, params, params["noise"])
    cond = float(spla.eigsh(K, k=1, which="LA", return_eigenvectors=False, tol=1e-4)[0]) / (params["noise"] + 1e-6)
    tol = RTOL * max(1.0, cond / 1e5)
    theta = theta_of(params, d)[None]
    for k, P in enumerate((40, 700, 3)):                                # 700 grows the buffer around the cached factor
        ctx.set_option("ozaki", first if k == 0 else later)
        Xn = rng.uniform(0, 1, (P, d))
        out, c = counted(ctx, lambda: ctx.posterior("Matern", X, y, Xn, theta, want=("mean", "var", "cov")))
        rmean, rcov = oracle.exact_posterior_chol(X, y, Xn, params, "Matern")
        check_posterior(out, rmean, rcov, tol, f"{seq} call {k} P={P} cond(K) <= {cond:.1e}")
        assert ctx.cache_hits() == k, (seq, k)                          # the toggle keeps the factor: it is the same matrix
        if k == 0:
            assert c["potrf_tall"] == (1 if first else 0) and c["potrf_diag"] == -(-N // 128), c
            continue
        assert c["potrf_diag"] == c["potrf_tall"] == c["panel_solve"] == 0, c      # nothing was factored again
        if seq == "all_int8":
            assert c["trsm_tall"] == 1 and c["oz_mma"] >= -(-N // 1024), c
        else:
            assert c["trsm_tall"] == 0, c                               # no kept inverses (fp64 factor) or int8 switched off
        if later == 0:
            assert c["oz_mma"] == c["oz_slice"] == 0, c                 # ozaki = 0 means fp64 only, cached int8 factor or not


# ------------------------------------------------------------------ 4. factorisation and solves under an explicit option
@pytest.mark.parametrize("ozaki", [0, 7])
@pytest.mark.parametrize("n", [2048, 4100])
def test_potrf_under_named_option(ctx, n, ozaki):
    rng = np.random.default_rng(n)
    A = spd(rng, n)
    ctx.set_option("ozaki", ozaki)
    (L, info), c = counted(ctx, lambda: ctx.potrf(A))
    assert info == 0
    Lt = np.tril(L)
    assert np.linalg.norm(Lt @ Lt.T - A) / np.linalg.norm(A) <= 1e-14 * n ** 0.5
    ref = sla.cholesky(A, lower=True)
    np.testing.assert_allclose(Lt, ref, rtol=0, atol=1e-10 * np.abs(ref).max())
    np.testing.assert_array_equal(np.triu(L, 1), np.triu(A, 1))                # strict upper untouched
    assert c["potrf_diag"] == -(-n // 128), c
    if ozaki == 0:
        assert c["potrf_tall"] == c["panel_solve"] == c["oz_mma"] == 0 and c["trsm_strip"] > 0, c
    else:
        # every diagonal block but the last has rows below it to solve
        assert c["potrf_tall"] == 1 and c["panel_solve"] == -(-n // 1024) - 1 and c["oz_mma"] >= c["panel_solve"], c


def leaf_rows_past_one_wave(sm):
    """rows of an in-place leaf solve that give more 128-row tiles than SMs and a partial last wave"""
    return 128 * (sm + 1) + 37


@pytest.mark.parametrize("ozaki", [0, 7])
@pytest.mark.parametrize("n,nrhs", [(2048, 300), (1536, 1025), (100, 14400), (100, None)])
def test_trsm_lower_under_named_option(ctx, n, nrhs, ozaki):
    """(100, 14400) is the in-place leaf solve (C aliases A, one column tile) with enough row tiles for the persistent TMA
    kernel; (100, None) has more row tiles than SMs plus a partial last wave, where that kernel hands the remainder to a
    follow-up launch: with C aliasing A each row block must still be read and written by one CTA only"""
    sm = ctx.device_info()["sm_count"]
    if nrhs is None:
        nrhs = leaf_rows_past_one_wave(sm)
    rng = np.random.default_rng(n + nrhs)
    A = spd(rng, n)
    B = rng.standard_normal((nrhs, n))
    ctx.set_option("ozaki", ozaki)
    L, info = ctx.potrf(A)
    assert info == 0
    X, c = counted(ctx, lambda: ctx.trsm_lower(L, B))
    ref = sla.solve_triangular(np.tril(L), B.T, lower=True).T
    np.testing.assert_allclose(X, ref, rtol=0, atol=1e-11 * np.abs(ref).max())
    if n == 100:
        # the leaf: X = B Linv^T is one GEMM; error like a DGEMM's, far below the solve's bar
        assert c["gemm_tma"] == 1 and c["gemm_nt"] == 0 and c["oz_mma"] == c["trsm_strip"] == 0, c
        np.testing.assert_allclose(X, ref, rtol=0, atol=1e-12 * np.abs(ref).max())
    elif ozaki == 0 or nrhs < 1024:
        assert c["panel_solve"] == c["oz_mma"] == 0 and c["trsm_strip"] > 0, c
    else:
        # >= 1024 rows against factor blocks of <= `panel` columns: 1536 splits into two 768-wide panel solves
        assert c["panel_solve"] == 2 and c["oz_mma"] == 2, c


# ------------------------------------------------------------------ 5. GEMM dispatch boundaries
def dgemm_scale(A, B, C0, ref):
    return np.linalg.norm(A, axis=1)[:, None] * np.linalg.norm(B, axis=1)[None, :] + np.abs(C0) + np.abs(ref)


@pytest.mark.parametrize("beta", [0.0, 1.0])
@pytest.mark.parametrize("k", [511, 512])
@pytest.mark.parametrize("short", [1, 0])
def test_int8_dispatch_boundary(ctx, short, k, beta):
    """with ozaki = 7 a product goes to the int8 kernel exactly when beta == 1, k >= 512 and it has at least
    `oz_min_tiles` (= the SM count) tiles of 128 x 64; one tile fewer, one k fewer or beta = 0 stays on fp64"""
    sm = ctx.device_info()["sm_count"]
    tiles = sm - short
    m, n = 128 * tiles, 64
    rng = np.random.default_rng(tiles + k)
    A, B, C0 = rng.standard_normal((m, k)), rng.standard_normal((n, k)), rng.standard_normal((m, n))
    ctx.set_option("ozaki", 7)
    assert ctx.get_option("oz_min_tiles") == sm
    C, c = counted(ctx, lambda: ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=beta))
    ref = beta * C0 - A @ B.T
    err = (np.abs(C - ref) / dgemm_scale(A, B, beta * C0, ref)).max()
    int8 = beta == 1.0 and k >= 512 and tiles >= sm
    assert (c["oz_mma"], c["oz_slice"]) == ((1, 2) if int8 else (0, 0)), c
    assert (c["gemm_nt"] + c["gemm_tma"] > 0) == (not int8), c
    assert err <= (2e-14 if int8 else 3e-15), err


# ------------------------------------------------------------------ 6. int8 kernel edges, bit for bit
def _rows(rng, m, k):
    return rng.standard_normal((m, k)) * np.exp(rng.normal(0, 2, (m, 1)))      # rows of very different scale


def int8_case(name, sm):
    """(A, B, C0, lower_only, int8 launches, oz_min_tiles or None): at least `sm` tiles of 128 x 64, so that the public GEMM
    hands the product to the int8 kernel under the default threshold -- except the long-k case, which lowers the threshold
    instead to keep the restatement's digit planes (S x rows x k int64) small"""
    rng = np.random.default_rng(sum(map(ord, name)))
    sq = next(s for s in range(1, 10 ** 4) if s * (s + 1) >= sm)        # lower-only tile count of an n x n update
    if name == "lower_square":
        n = 128 * sq - 36
        A = _rows(rng, n, 555)
        return A, A, rng.standard_normal((n, n)), True, 1, None
    if name == "lower_trapezoid":
        n = 128 * sq - 36
        A = _rows(rng, n + 700, 600)                                    # k not a multiple of 32
        return A, A[:n], rng.standard_normal((n + 700, n)), True, 1, None
    if name == "k_split":
        m, n, k = 384, 128, oz.K_MAX + 96                               # two launches, the second with k = 96
        return _rows(rng, m, k), _rows(rng, n, k), rng.standard_normal((m, n)), False, 2, 6
    if name == "odd_column_tiles":
        m, n, k = 128 * -(-sm // 3) + 5, 190, 520                       # 3 column tiles: a CTA pair with one column tile idle
        return _rows(rng, m, k), _rows(rng, n, k), rng.standard_normal((m, n)), False, 1, None
    if name in ("single_column_tile", "zero_and_extreme_rows"):
        m, n, k = 128 * sm, 50, 512
        A, B = _rows(rng, m, k), _rows(rng, n, k)
        if name == "zero_and_extreme_rows":
            A[3] = 0.0
            B[2] = 0.0
            A[5] *= 2.0 ** 200
            A[130] *= 2.0 ** -200
            B[1] *= 2.0 ** -200
            B[7] *= 2.0 ** 200
        return A, B, rng.standard_normal((m, n)), False, 1, None
    raise KeyError(name)


@pytest.mark.parametrize("S", [7, 6])
@pytest.mark.parametrize("name", ["lower_square", "lower_trapezoid", "k_split", "odd_column_tiles", "single_column_tile",
                                  "zero_and_extreme_rows"])
def test_int8_kernel_edges_equal_the_restatement_bit_for_bit(ctx, name, S):
    """exact integer products and the same fixed-order fp64 recombination on both sides -> identical doubles, as CTA pairs
    (oz_cluster = 2) and as independent CTAs (1)"""
    A, B, C0, lower, launches, min_tiles = int8_case(name, ctx.device_info()["sm_count"])
    if min_tiles is not None:
        ctx.set_option("oz_min_tiles", min_tiles)
    want = oz.gemm_nt(A, B, C0, alpha=-1.0, S=S, lower_only=lower)
    ctx.set_option("ozaki", S)
    got = {}
    for cl in (2, 1):
        ctx.set_option("oz_cluster", cl)
        got[cl], c = counted(ctx, lambda: ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0, lower_only=lower))
        assert c["oz_mma"] == launches and c["gemm_nt"] == c["gemm_tma"] == 0, (cl, c)
        np.testing.assert_array_equal(got[cl], want, err_msg=f"{name} S={S} oz_cluster={cl}")
    np.testing.assert_array_equal(got[1], got[2])
    if lower:
        n = C0.shape[1]
        np.testing.assert_array_equal(np.triu(got[2][:n], 1), np.triu(C0[:n], 1))   # strict upper of the square part untouched


def test_lower_only_trapezoid_on_the_fp64_kernels(ctx):
    """m > n with lower_only through the public entry point at ozaki = 0: the square part on the triangular tile map,
    the rows below it as a plain product"""
    A, B, C0, _, _, _ = int8_case("lower_trapezoid", ctx.device_info()["sm_count"])
    m, n = C0.shape
    assert ctx.get_option("ozaki") == 0
    C, c = counted(ctx, lambda: ctx.gemm_nt(A, B, C0, alpha=-1.0, beta=1.0, lower_only=True))
    assert c["oz_mma"] == 0 and c["gemm_nt"] + c["gemm_tma"] >= 2, c
    ref = C0 - A @ B.T
    mask = np.tril(np.ones((m, n), bool))
    assert (np.abs(C - ref) / dgemm_scale(A, B, C0, ref))[mask].max() <= 3e-15
    np.testing.assert_array_equal(C[~mask], C0[~mask])
    from gpax_b200._ffi import B200GPError
    with pytest.raises(B200GPError):                                    # fewer rows than columns has no lower trapezoid
        ctx.gemm_nt(A[:n - 1], B, C0[:n - 1], alpha=-1.0, beta=1.0, lower_only=True)


# ------------------------------------------------------------------ 7. panel-solve modes of the int8 kernel
@pytest.mark.parametrize("n", [1024, 1000, 520])
def test_panel_solve_through_the_int8_kernel(ctx, n):
    """>= 1024 right-hand sides against a factor of at most `panel` columns: one panel_solve_all_rows, i.e. the int8 kernel
    in its overwrite + transposed-B + k-triangular mode with C aliasing A's storage"""
    nrhs = 1500
    rng = np.random.default_rng(n)
    A = spd(rng, n)
    B = rng.standard_normal((nrhs, n))
    res = {}
    for ozaki in (0, 7):
        ctx.set_option("ozaki", ozaki)
        L, info = ctx.potrf(A)
        assert info == 0
        X, c = counted(ctx, lambda: ctx.trsm_lower(L, B))
        assert (c["panel_solve"], c["oz_mma"]) == ((1, 1) if ozaki else (0, 0)), (ozaki, c)
        ref = sla.solve_triangular(np.tril(L), B.T, lower=True).T
        np.testing.assert_allclose(X, ref, rtol=0, atol=1e-11 * np.abs(ref).max())
        res[ozaki] = X
    assert not np.array_equal(res[7], res[0])
    np.testing.assert_allclose(res[7], res[0], rtol=0, atol=1e-12 * np.abs(res[0]).max())


# ------------------------------------------------------------------ 8. multi-GPU entry point with default options
def test_dist_posterior_works_on_a_context_with_default_options(ctx):
    """DistContext.posterior on a context nobody set an option on (1 x 1 grid): the block-cyclic factorisation has no fp64
    trailing update, so the default ozaki = 0 picks the digit planes from the conditioning bound like -1 does"""
    from dist_lib_worker import problem as dist_problem
    from test_gpu_dist_lib import TOL, run_grid
    N, P, nb, kernel = 2048, 300, 256, "Matern"
    assert "B200GP_TEST_OZAKI" not in os.environ
    res = run_grid(1, 1, N, P, nb, kernel, ozaki=None)[0]
    assert res["info"] == 0 and res["ozaki"] == 0                       # the worker set no option
    X, y, Xn, theta = dist_problem(N, P, kernel)
    with ctx.options(ozaki=-1):
        ref = ctx.posterior(kernel, X, y, Xn, theta[None], want=("mean", "var"))
    assert_close(res["mean"], ref["mean"][0], TOL[-1], "mean, 1 x 1 grid, default options")
    assert_close(res["var"], ref["var"][0], TOL[-1], "var, 1 x 1 grid, default options")
