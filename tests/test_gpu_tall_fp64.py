"""GPU: the tall-panel factorisation on the fp64 DMMA route (ozaki = 0, panel > 0, N >= tall_min_fp64).

Each diagonal block's panel solve is one in-place k-triangular DMMA GEMM over every row below the block, the test-point
rows [k_pX; y^T] included (gemm_panel_solve, potrf.cuh).  As in test_gpu_paths.py each test sets its options on a context
of its own and asserts the numbers and the route (Context.path_counts()) together."""
import functools

import numpy as np
import pytest
import scipy.sparse.linalg as spla

import oracle
from conftest import assert_close

pytestmark = pytest.mark.gpu

RTOL = 1e-9   # the parity bar at cond(K) <= 1e5, scaled by cond / 1e5 beyond (as in test_gpu_paths.py)
PARAMS = {"k_length": np.array([0.25, 0.35]), "k_scale": 1.1, "noise": 0.05, "period": 0.9}


@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def counted(ctx, fn):
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


def theta_of(params, d):
    ell = np.broadcast_to(np.asarray(params["k_length"], dtype=float).reshape(-1), (d,))
    return np.concatenate([ell, [params["k_scale"], params["noise"], params.get("period", 1.0)]])


@functools.lru_cache(maxsize=2)
def problem(kname, N, P):
    rng = np.random.default_rng(N + 7 * P)
    d = 2
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    rmean, rcov = oracle.exact_posterior_chol(X, y, Xn, PARAMS, kname)
    K = oracle.get_kernel(kname)(X, X, PARAMS, PARAMS["noise"])
    cond = float(spla.eigsh(K, k=1, which="LA", return_eigenvectors=False, tol=1e-4)[0]) / (PARAMS["noise"] + 1e-6)
    return X, y, Xn, rmean, rcov, RTOL * max(1.0, cond / 1e5), cond


def check(out, rmean, rcov, tol, what, cov=True):
    assert out["info"][0] == 0, what
    assert_close(out["mean"][0], rmean, tol, "mean " + what)
    assert_close(out["var"][0], np.diag(rcov), tol, "var " + what)
    if cov:
        assert_close(out["cov"][0], rcov, tol, "cov " + what)


def assert_fp64_tall(c, N, panel):
    assert c["potrf_tall_fp64"] == 1 and c["panel_solve"] == -(-N // panel), c
    assert c["oz_mma"] == c["oz_slice"] == c["potrf_tall"] == c["trsm_tall"] == 0, c
    assert c["potrf_diag"] == -(-N // 128), c


def test_default_threshold_ragged_N_vs_oracle(ctx):
    """N = 8300 (last panel 108 wide) under the shipped options; P + 1 = 1001 test-point rows, not a multiple of 128"""
    N, P, kname = 8300, 1000, "Matern"
    assert (ctx.get_option("ozaki"), ctx.get_option("panel")) == (0, 1024)
    assert 4100 < ctx.get_option("tall_min_fp64") <= N
    X, y, Xn, rmean, rcov, tol, cond = problem(kname, N, P)
    out, c = counted(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta_of(PARAMS, 2)[None], want=("mean", "var", "cov")))
    check(out, rmean, rcov, tol, f"N={N} cond(K) <= {cond:.1e}")
    assert_fp64_tall(c, N, 1024)
    assert c["trsm_strip"] > 0, c          # only inside the diagonal blocks (U = L_bb^{-T})


@pytest.mark.parametrize("panel", [256, 512, 1024])
@pytest.mark.parametrize("N,P", [(2500, 300), (3100, 47)])
def test_lowered_threshold_over_panel_widths(ctx, N, P, panel):
    """below the default threshold with tall_min_fp64 lowered: every panel width, ragged N, P + 1 rows not a multiple of
    128, and row counts that leave a partial last wave of row strips"""
    kname = "RBF" if N == 2500 else "Periodic"
    X, y, Xn, rmean, rcov, tol, cond = problem(kname, N, P)
    with ctx.options(tall_min_fp64=2048, panel=panel):
        out, c = counted(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta_of(PARAMS, 2)[None], want=("mean", "var", "cov")))
    check(out, rmean, rcov, tol, f"N={N} P={P} panel={panel} cond(K) <= {cond:.1e}")
    assert_fp64_tall(c, N, panel)


@pytest.mark.parametrize("n", [4100, 8300])
def test_potrf_reconstructs_on_the_fp64_tall_route(ctx, n):
    rng = np.random.default_rng(n)
    X = rng.uniform(0, 1, (n, 2))
    A = oracle.get_kernel("Matern")(X, X, PARAMS, PARAMS["noise"])
    with ctx.options(tall_min_fp64=2048):
        (L, info), c = counted(ctx, lambda: ctx.potrf(A))
    assert info == 0
    Lt = np.tril(L)
    V = rng.standard_normal((n, 8))
    err = np.linalg.norm(Lt @ (Lt.T @ V) - A @ V) / np.linalg.norm(A @ V)
    assert err <= 1e-14 * n ** 0.5, err
    np.testing.assert_array_equal(np.triu(L, 1), np.triu(A, 1))                # strict upper untouched
    assert c["potrf_tall_fp64"] == 1 and c["panel_solve"] == -(-n // 1024) - 1, c    # the last block has no rows below
    assert c["oz_mma"] == c["oz_slice"] == c["potrf_tall"] == 0, c


def test_posterior_grad_mean_var_bit_identical_to_posterior(ctx):
    """the headline shape: P d derivative rows ride in the factorisation too (4097 right-hand-side rows, more 128-row
    strips than SMs in the first panel solves), and mean / var keep the bits of b2gp_posterior"""
    N, P, d = 16384, 1024, 3
    rng = np.random.default_rng(5)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(3 * X[:, 0]) * np.cos(2 * X[:, 1]) + X[:, 2] + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    theta = np.array([[0.3, 0.32, 0.28, 1.0, 0.1, 1.0]])
    plain, c1 = counted(ctx, lambda: ctx.posterior("RBF", X, y, Xn, theta, want=("mean", "var")))
    ctx.set_option("drop_factor_cache", 1)
    grad, c2 = counted(ctx, lambda: ctx.posterior_grad("RBF", X, y, Xn, theta))
    for c in (c1, c2):
        assert_fp64_tall(c, N, 1024)
        assert c["gemm_tma"] > 0, c
    assert plain["info"][0] == 0 and grad["info"][0] == 0
    assert np.array_equal(grad["mean"], plain["mean"])
    assert np.array_equal(grad["var"], plain["var"])
    assert np.isfinite(grad["dmean"]).all() and np.isfinite(grad["dvar"]).all()


def test_fp64_tall_factor_then_int8_cache_hit(ctx):
    """an fp64-tall factor keeps no explicit block inverses, so an ozaki = 7 call that reuses it solves by trsm_rec"""
    N, P, kname = 8300, 1000, "Matern"
    X, y, Xn, rmean, rcov, tol, cond = problem(kname, N, P)
    theta = theta_of(PARAMS, 2)[None]
    out, c = counted(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta, want=("mean", "var")))
    check(out, rmean, rcov, tol, "fp64-tall factor", cov=False)
    assert_fp64_tall(c, N, 1024)
    ctx.set_option("ozaki", 7)
    out, c = counted(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta, want=("mean", "var", "cov")))
    assert ctx.cache_hits() == 1
    check(out, rmean, rcov, tol, f"ozaki=7 cache hit on the fp64-tall factor, cond(K) <= {cond:.1e}")
    assert c["potrf_diag"] == c["potrf_tall"] == c["potrf_tall_fp64"] == c["trsm_tall"] == 0, c


def test_panel_zero_is_the_recursive_route_bit_for_bit(ctx):
    """panel = 0 leaves the recursive scheme (potrf_rec, then trsm_rec of the test-point rows) exactly as it was"""
    N, P, kname = 8300, 1000, "Matern"
    X, y, Xn, rmean, rcov, tol, cond = problem(kname, N, P)
    theta = theta_of(PARAMS, 2)[None]
    with ctx.options(panel=0):
        a, ca = counted(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta, want=("mean", "var")))
    with ctx.options(tall_min_fp64=1 << 30):
        b, cb = counted(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta, want=("mean", "var")))
    for c in (ca, cb):
        assert c["potrf_tall_fp64"] == c["panel_solve"] == c["potrf_tall"] == c["oz_mma"] == 0 and c["trsm_strip"] > 0, c
    assert np.array_equal(a["mean"], b["mean"]) and np.array_equal(a["var"], b["var"])
    check(a, rmean, rcov, tol, "panel=0", cov=False)
