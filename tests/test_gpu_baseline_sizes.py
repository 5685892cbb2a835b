"""GPU: the CUDA path against the ORACLE at BASELINE.json's own sizes (SURVEY.md section 8d rows), not only through
size-independent properties:

  headline  N=16384 d=3 P=1024 RBF          vs oracle.exact_posterior_chol, int8 wgmma path (auto / 7 / 6 planes) and fp64 DMMA
  C2        N=8192 d=2 Matern, 200 draws    2 of the draws vs oracle.exact_posterior (explicit inverse, gp.py:271) + mean(0) wiring
  C3        N=16384 viGP (mean, var)         a 1000-point tile of the 181x181 grid vs the Cholesky oracle (vigp.py:178-185)
  sparse    cond(Kuu) <= 1e5 at 1e-9, and M=4096 / N=32768 (sparse_gp.py:173-223)

Every assertion message states the conditioning the 1e-9 bar is taken at (lambda_max by Lanczos over the oracle's own K,
lambda_min >= noise + jitter).  The oracle costs ~10-30 s per case on the GPU box's host cores.
"""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import oracle
from conftest import assert_close

pytestmark = pytest.mark.gpu
RTOL = 1e-9


@pytest.fixture(scope="module")
def ctx():
    import gpax_b200
    c = gpax_b200.default_context()
    with c.options(ozaki=c.get_option("ozaki"), streams=c.get_option("streams")):      # whatever a test sets is put back
        yield c


def cond_bound(K, floor):
    """lambda_max(K) (Lanczos) / floor, floor = noise + jitter <= lambda_min(K) for K = k(X,X) + (noise + jitter) I"""
    lam = spla.eigsh(K, k=1, which="LA", return_eigenvectors=False, tol=1e-4)[0]
    return float(lam / floor)


def headline_inputs():
    N, d, P = 16384, 3, 1024
    rng = np.random.default_rng(4)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(3 * X[:, 0]) * np.cos(2 * X[:, 1]) + X[:, 2] + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    params = {"k_length": np.full(d, 0.3), "k_scale": 1.0, "noise": 0.1}
    return X, y, Xn, params


def test_headline_N16384_vs_oracle(ctx):
    """The benchmark workload itself (bench.py WORKLOAD) against the Cholesky oracle: mean, diag variance and the full
    P x P covariance, through the int8 wgmma path at every plane setting and through the all-fp64 DMMA path."""
    X, y, Xn, params = headline_inputs()
    d = X.shape[1]
    K = oracle.rbf_kernel(X, X, params, params["noise"], jitter=1e-6)
    cond = cond_bound(K, params["noise"] + 1e-6)
    del K
    rmean, rcov = oracle.exact_posterior_chol(X, y, Xn, params, "RBF")
    rvar = rcov.diagonal()
    theta = np.concatenate([params["k_length"], [1.0, 0.1, 1.0]])[None, :]
    tol = RTOL * max(1.0, cond / 1e5)
    for planes in (-1, 7, 6, 0):
        want = ("mean", "var", "cov") if planes in (-1, 0) else ("mean", "var")      # full covariance on the default path too
        with ctx.options(ozaki=planes):
            ctx.set_option("drop_factor_cache", 1)
            before = ctx.path_counts()
            out = ctx.posterior("RBF", X, y, Xn, theta, want=want)
            moved = {k: v - before[k] for k, v in ctx.path_counts().items()}
        assert out["info"][0] == 0
        assert (moved["oz_mma"] > 0) == (moved["potrf_tall"] == 1) == (planes != 0), (planes, moved)
        what = f"N=16384 headline, ozaki={planes}, cond(K) <= {cond:.2e}"
        # 6 digit planes are what the auto rule picks below cond 1e6 (DESIGN 4.6); when forced above that they get the
        # model's bound instead of the parity bar
        t = tol if planes != 6 or cond <= 1e6 else tol * cond / 1e6
        assert_close(out["mean"][0], rmean, t, "mean " + what)
        assert_close(out["var"][0], rvar, t, "var " + what)
        err_m = np.abs(out["mean"][0] - rmean).max() / np.abs(rmean).max()
        err_v = np.abs(out["var"][0] - rvar).max() / np.abs(rvar).max()
        print(f"{what}: scaled error mean {err_m:.2e} var {err_v:.2e}")
        if "cov" in want:
            assert_close(out["cov"][0], rcov, t, "cov " + what)


def c2_inputs():
    """SURVEY 8d row C2: N=8192 d=2 U(0,1)^2 seed 1, Matern, S=200 draws seed 2, P=1024."""
    N, d, P, S = 8192, 2, 1024, 200
    rng = np.random.default_rng(1)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(4 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    r2 = np.random.default_rng(2)
    samples = {"k_length": np.exp(r2.normal(np.log(0.3), 0.1, (S, d))), "k_scale": np.exp(r2.normal(0.0, 0.1, S)),
               "noise": np.exp(r2.normal(np.log(0.1), 0.1, S))}
    return X, y, Xn, samples


def test_c2_N8192_200_draws_vs_oracle():
    """ExactGP.predict over the 200 draws (gp.py:351-399): two of the draws against the explicit-inverse oracle, and the
    y_means.mean(0) wiring of gp.py:393-399 against the per-draw means of a second, separate call."""
    import gpax_b200
    X, y, Xn, samples = c2_inputs()
    S = len(samples["noise"])
    m = gpax_b200.ExactGP(2, "Matern")
    m.X_train, m.y_train = X, y
    streams0 = m.ctx.get_option("streams")
    m.ctx.set_option("streams", 4)
    mean, y_sampled = m.predict(0, Xn, samples, n=1)
    assert mean.shape == (1024,) and y_sampled.shape == (S, 1, 1024) and np.isfinite(y_sampled).all()
    theta = np.column_stack([samples["k_length"], samples["k_scale"], samples["noise"], np.ones(S)])
    per_draw = m.ctx.posterior("Matern", X, y, Xn, theta, want=("mean", "var"))
    assert (per_draw["info"] == 0).all()
    np.testing.assert_allclose(mean, per_draw["mean"].mean(0), rtol=1e-13, atol=1e-13)
    for s in (0, 137):
        ps = {k: v[s] for k, v in samples.items()}
        K = oracle.matern_kernel(X, X, ps, ps["noise"], jitter=1e-6)
        cond = cond_bound(K, ps["noise"] + 1e-6)
        del K
        rmean, rcov = oracle.exact_posterior(X, y, Xn, ps, "Matern")
        tol = RTOL * max(1.0, cond / 1e5)
        what = f"C2 draw {s}: N=8192 Matern, cond(K) <= {cond:.2e}"
        assert_close(per_draw["mean"][s], rmean, tol, "mean " + what)
        assert_close(per_draw["var"][s], rcov.diagonal(), tol, "var " + what)
        one = m.get_mvn_posterior(Xn, ps)
        assert_close(one[0], rmean, tol, "get_mvn_posterior mean " + what)
        assert_close(one[1], rcov, tol, "get_mvn_posterior cov " + what)
    m.ctx.set_option("streams", streams0)


def test_c3_N16384_vigp_tile_vs_oracle():
    """SURVEY 8d row C3: 16384 random pixels of a 181x181 grid, Matern l=[4.2, 3.2], scale 0.05, noise 0.002; viGP.predict
    (mean, var) on a 1000-point tile of the full grid against the Cholesky oracle of vigp.py:178-185."""
    import gpax_b200
    n = 181
    rng = np.random.default_rng(3)
    gx, gy = np.meshgrid(np.arange(n, dtype=float), np.arange(n, dtype=float), indexing="ij")
    full = np.column_stack([gx.ravel(), gy.ravel()])
    idx = rng.choice(n * n, 16384, replace=False)
    X = full[idx]
    f = np.sin(X[:, 0] / 17.0) * np.cos(X[:, 1] / 23.0) + 0.3 * np.sin((X[:, 0] + X[:, 1]) / 9.0)
    y = (f - f.min()) / (f.max() - f.min()) + 0.02 * rng.standard_normal(len(X))
    params = {"k_length": np.array([4.2, 3.2]), "k_scale": 0.05, "noise": 0.002}
    tile = full[7000:8000]
    K = oracle.matern_kernel(X, X, params, params["noise"], jitter=1e-6)
    cond = cond_bound(K, params["noise"] + 1e-6)
    del K
    rmean, rvar = oracle.exact_posterior_chol(X, y, tile, params, "Matern", noiseless=True, diag_only=True)
    v = gpax_b200.viGP(2, "Matern")
    v.X_train, v.y_train = X, y
    mean, var = v.predict(None, tile, samples=params, noiseless=True)
    tol = RTOL * max(1.0, cond / 1e5)
    what = f"C3 N=16384 viGP tile, cond(K) <= {cond:.2e}"
    assert_close(mean, rmean, tol, "mean " + what)
    assert_close(var, rvar, tol, "var " + what)
    # the chunked entry point re-uses the factor (33 chunks in the reference's setting; 4 here)
    mb, vb = v.predict_in_batches(None, tile, batch_size=250, samples=params, noiseless=True)
    assert_close(mb, rmean, tol, "batched mean " + what)
    assert_close(vb, rvar, tol, "batched var " + what)


def test_sparse_well_conditioned_1e9():
    """viSparseGP.get_mvn_posterior with cond(Kuu) ~ 4e1: the 1e-9 bar with no conditioning allowance."""
    import gpax_b200
    rng = np.random.default_rng(11)
    N, P = 3000, 300
    g = np.linspace(0.05, 0.95, 8)
    Xu = np.array([[a, b] for a in g for b in g])
    X = rng.uniform(0, 1, (N, 2))
    y = np.sin(5 * X[:, 0]) * np.cos(4 * X[:, 1]) + 0.05 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, 2))
    params = {"k_length": np.array([0.12, 0.12]), "k_scale": 1.0, "noise": 0.05}
    cond = np.linalg.cond(oracle.matern_kernel(Xu, Xu, params, jitter=1e-5))
    assert cond <= 1e5
    m = gpax_b200.viSparseGP(2, "Matern")
    m.X_train, m.y_train, m.Xu = X, y, Xu
    for nl in (False, True):
        rmean, rcov = oracle.sparse_posterior(X, y, Xu, Xn, params, "Matern", noiseless=nl, jitter=1e-5)
        mean, cov = m.get_mvn_posterior(Xn, params, noiseless=nl, jitter=1e-5)
        what = f"sparse N={N} M=64, cond(Kuu) = {cond:.1e}"
        assert_close(mean, rmean, RTOL, "mean " + what)
        assert_close(cov, rcov, RTOL, "cov " + what)


def test_sparse_M4096_N32768_vs_oracle(ctx):
    """C5's inducing-set size on one GPU: M=4096 (64x64 grid), N=32768, P=512, Matern l=0.03 (cond(Kuu) ~ 4e3)."""
    rng = np.random.default_rng(6)
    N, P = 32768, 512
    g = (np.arange(64) + 0.5) / 64
    Xu = np.array([[a, b] for a in g for b in g])
    X = rng.uniform(0, 1, (N, 2))
    y = np.sin(9 * X[:, 0]) * np.cos(7 * X[:, 1]) + 0.05 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, 2))
    params = {"k_length": np.array([0.03, 0.03]), "k_scale": 1.0, "noise": 0.05}
    Kuu = oracle.matern_kernel(Xu, Xu, params, jitter=1e-5)
    w = np.linalg.eigvalsh(Kuu)
    cond = float(w[-1] / w[0])
    del Kuu
    rmean, rcov = oracle.sparse_posterior(X, y, Xu, Xn, params, "Matern", jitter=1e-5)
    theta = np.array([0.03, 0.03, 1.0, 0.05, 1.0])
    out = ctx.sparse_posterior("Matern", Xu, X, y, Xn, theta, jitter=1e-5, want=("mean", "var", "cov"))
    assert out["info"] == 0
    tol = RTOL * max(1.0, cond / 1e5)
    what = f"sparse N={N} M=4096, cond(Kuu) = {cond:.1e}"
    assert_close(out["mean"], rmean, tol, "mean " + what)
    assert_close(out["cov"], rcov, tol, "cov " + what)
    assert_close(out["var"], rcov.diagonal(), tol, "var " + what)
