"""GPU: the posterior path through the C-ABI and the Python shell, against the golden vectors
(reference source) and the oracle; plus the reference's behavioural test contract (SURVEY.md section 4)."""
import numpy as np
import pytest

import oracle
from conftest import assert_close

pytestmark = pytest.mark.gpu

RTOL = 1e-9   # BASELINE.json: predict-path outputs within 1e-9 rtol (scale-relative atol, cond(K) <= 1e5)


@pytest.fixture(scope="module")
def gp():
    import gpax_b200
    return gpax_b200


def theta_of(params, d):
    ell = np.broadcast_to(np.asarray(params["k_length"], dtype=float).reshape(-1), (d,))
    return np.concatenate([ell, [params["k_scale"], params["noise"], params.get("period", 1.0)]])


# ------------------------------------------------------------------ golden vectors (reference source)
@pytest.mark.parametrize("kname", ["RBF", "Matern", "Periodic"])
def test_exact8_golden(gp, golden, kname):
    """the reference's own test setting (tests/test_gp.py:139-152) with seeded data"""
    m = gp.ExactGP(1, kernel=kname)
    m.X_train, m.y_train = golden["exact8_Xtr"], golden["exact8_ytr"]
    params = {"k_length": np.array([1.0]), "k_scale": 1.0, "noise": 0.1, "period": 1.0}
    K = oracle.get_kernel(kname)(golden["exact8_Xtr"][:, None], golden["exact8_Xtr"][:, None], params, 0.1)
    cond = np.linalg.cond(K)
    # the bar is 1e-9 for cond <= 1e5; beyond that the LU-inverse reference loses digits itself (SURVEY fact 9)
    rtol = RTOL * max(1.0, cond / 1e5)
    for nl in (0, 1):
        mean, cov = m.get_mvn_posterior(golden["exact8_Xte"], params, noiseless=bool(nl))
        assert mean.shape == (20,) and cov.shape == (20, 20)
        assert_close(mean, golden[f"exact8_{kname}_nl{nl}_mean"], rtol, f"mean cond={cond:.1e}")
        assert_close(cov, golden[f"exact8_{kname}_nl{nl}_cov"], rtol, f"cov cond={cond:.1e}")
    mean, cov = m.get_mvn_posterior(golden["exact8_Xte"], params, jitter=1e-5)
    assert_close(mean, golden[f"exact8_{kname}_jit1e-5_mean"], rtol)
    assert_close(cov, golden[f"exact8_{kname}_jit1e-5_cov"], rtol)


@pytest.mark.parametrize("kname,N", [("RBF", 300), ("Matern", 384), ("Periodic", 200)])
def test_exact_medium_golden(gp, golden, kname, N):
    tag = f"exact_{kname}_N{N}"
    Xtr, ytr, Xte, ell = (golden[tag + s] for s in ("_Xtr", "_ytr", "_Xte", "_ell"))
    params = {"k_length": ell, "k_scale": 1.2, "noise": 0.1, "period": 0.8}
    m = gp.ExactGP(Xtr.shape[1], kernel=kname)
    m.X_train, m.y_train = Xtr, ytr
    mean, cov = m.get_mvn_posterior(Xte, params)
    assert_close(mean, golden[tag + "_mean"], RTOL)
    assert_close(cov, golden[tag + "_cov"], RTOL)
    assert np.array_equal(cov, cov.T)
    v = gp.viGP(Xtr.shape[1], kernel=kname)
    v.X_train, v.y_train = Xtr, ytr
    vm, vv = v.predict(None, Xte, samples=params, noiseless=True)
    assert_close(vm, golden[tag + "_vimean"], RTOL)
    assert_close(vv, golden[tag + "_vivar"], RTOL)


def test_mean_fn_golden(gp, golden):
    mfn = lambda x, p: p["a"] * x[:, 0] ** 2 + p["b"]   # noqa: E731
    m = gp.ExactGP(1, "RBF", mean_fn=mfn, mean_fn_prior=lambda: None)
    m.X_train, m.y_train = golden["meanfn_Xtr"], golden["meanfn_ytr"]
    params = {"k_length": np.array([0.5]), "k_scale": 1.0, "noise": 0.05, "a": 9.0, "b": 0.5}
    mean, cov = m.get_mvn_posterior(golden["meanfn_Xte"], params)
    assert_close(mean, golden["meanfn_mean"], RTOL)
    assert_close(cov, golden["meanfn_cov"], RTOL)


@pytest.mark.parametrize("tag,kname", [("sparse50", "RBF"), ("sparse400", "Matern")])
def test_sparse_golden(gp, golden, tag, kname):
    Xtr, ytr, Xu, Xte = (golden[tag + s] for s in ("_Xtr", "_ytr", "_Xu", "_Xte"))
    d = Xtr.shape[1]
    m = gp.viSparseGP(d, kernel=kname)
    m.X_train, m.y_train, m.Xu = Xtr, ytr, Xu
    params = {"k_length": np.full(d, 0.4), "k_scale": 1.0, "noise": 0.1}
    for nl in (0, 1):
        mean, cov = m.get_mvn_posterior(Xte, params, noiseless=bool(nl), jitter=1e-5)
        assert mean.shape == (25,) and cov.shape == (25, 25)
        # Kuu with jitter 1e-5 has cond ~1e6..1e9: both sides lose digits; tolerance scaled like above
        assert_close(mean, golden[f"{tag}_nl{nl}_mean"], 1e-6)
        assert_close(cov, golden[f"{tag}_nl{nl}_cov"], 1e-6)
    pm, pv = m.predict(None, Xte, samples=params, noiseless=True, jitter=1e-5)
    assert_close(pm, golden[f"{tag}_nl1_mean"], 1e-6)
    assert_close(pv, np.diag(golden[f"{tag}_nl1_cov"]), 1e-6)


# ------------------------------------------------------------------ oracle at larger sizes, all output kinds
@pytest.mark.parametrize("kname,N,P,d", [("RBF", 512, 1024, 1), ("Matern", 1000, 333, 2), ("RBF", 2048, 100, 3),
                                         ("Periodic", 700, 64, 1)])
def test_posterior_vs_oracle(gp, kname, N, P, d):
    """C1 of BASELINE.json is the first case: ExactGP RBF 1D N=512, single draw, fp64"""
    rng = np.random.default_rng(N + P)
    Xtr = rng.uniform(0, 1, (N, d))
    ytr = np.sin(6 * Xtr[:, 0]) + 0.1 * rng.standard_normal(N)
    Xte = np.linspace(0, 1, P)[:, None] if d == 1 else rng.uniform(0, 1, (P, d))
    params = {"k_length": np.full(d, 0.2 if d == 1 else 0.3), "k_scale": 1.0, "noise": 0.1, "period": 0.7}
    ref_mean, ref_cov = oracle.exact_posterior(Xtr, ytr, Xte, params, kname)
    ctx = gp.default_context()
    out = ctx.posterior(kname, Xtr, ytr, Xte, theta_of(params, d)[None], want=("mean", "var", "cov"), timing=True)
    assert out["info"][0] == 0
    assert_close(out["mean"][0], ref_mean, RTOL, "mean")
    assert_close(out["cov"][0], ref_cov, RTOL, "cov")
    assert_close(out["var"][0], np.diag(ref_cov), RTOL, "var")
    assert out["timing"]["total_ms"] > 0 and out["timing"]["launches"] > 0


def test_batched_draws_and_sampling(gp):
    """S draws in one call == S single-draw calls == oracle loop; samples = mean + chol(cov) eps"""
    rng = np.random.default_rng(7)
    N, P, d, S, n = 300, 40, 2, 5, 3
    Xtr, Xte = rng.uniform(0, 1, (N, d)), rng.uniform(0, 1, (P, d))
    ytr = np.sin(4 * Xtr[:, 0]) * np.cos(3 * Xtr[:, 1]) + 0.1 * rng.standard_normal(N)
    samples = {"k_length": np.exp(rng.normal(np.log(0.3), 0.1, (S, d))), "k_scale": np.exp(rng.normal(0, 0.1, S)),
               "noise": np.exp(rng.normal(np.log(0.1), 0.1, S))}
    eps = rng.standard_normal((S, n, P))
    ymean, means, ysamp = oracle.predict_draws(Xtr, ytr, Xte, samples, "Matern", n=n, eps=eps)
    theta = np.concatenate([samples["k_length"], samples["k_scale"][:, None], samples["noise"][:, None], np.ones((S, 1))], 1)
    ctx = gp.default_context()
    for streams in (1, 2, 4):
        with ctx.options(streams=streams):
            out = ctx.posterior("Matern", Xtr, ytr, Xte, theta, want=("mean", "cov"), eps=eps)
        assert_close(out["mean"], means, RTOL)
        assert_close(out["mean"].mean(0), ymean, RTOL)
        # chol(cov) amplifies rounding of cov by its condition number: looser bar on the samples
        assert_close(out["y_sampled"], ysamp, 1e-6)
    one = ctx.posterior("Matern", Xtr, ytr, Xte, theta[2:3], want=("mean", "cov"))
    np.testing.assert_array_equal(one["mean"][0], out["mean"][2])      # batched == single, bit for bit
    np.testing.assert_array_equal(one["cov"][0], out["cov"][2])


def test_non_pd_draw_gives_nan_not_exception(gp):
    """the reference's tests feed negative hyper-parameters (tests/test_gp.py:196-198); Cholesky cannot
    factor an indefinite K: that draw is NaN + info, the others are untouched"""
    rng = np.random.default_rng(1)
    N, P = 64, 10
    Xtr, Xte = rng.uniform(0, 1, (N, 1)), rng.uniform(0, 1, (P, 1))
    ytr = rng.standard_normal(N)
    theta = np.array([[0.3, 1.0, 0.1, 1.0], [0.3, -1.0, 0.1, 1.0], [0.3, 1.0, 0.1, 1.0]])
    out = gp.default_context().posterior("RBF", Xtr, ytr, Xte, theta, want=("mean", "var", "cov"),
                                         eps=rng.standard_normal((3, 2, P)))
    assert out["info"][0] == 0 and out["info"][2] == 0 and out["info"][1] > 0
    for k in ("mean", "var", "cov", "y_sampled"):
        assert np.isnan(out[k][1]).all() and np.isfinite(out[k][0]).all() and np.isfinite(out[k][2]).all()
    for k in ("mean", "var", "cov"):
        np.testing.assert_array_equal(out[k][0], out[k][2])      # same theta -> same bits, whatever ran in between


# ------------------------------------------------------------------ reference behavioural contract
def dummy(n=8, seed=0):
    rng = np.random.default_rng(seed)
    X = np.linspace(1, 2, n) + 0.1 * rng.standard_normal(n)
    return X, 10 * X ** 2


def test_get_mvn_posterior_contract(gp):
    """tests/test_gp.py:139-170: shapes, noiseless leaves the mean bit-identical, repeatability"""
    X, y = dummy()
    Xt = np.linspace(1, 2, 20)[:, None]
    params = {"k_length": np.array([1.0]), "k_scale": np.array(1.0), "noise": np.array(0.1)}
    m = gp.ExactGP(1, "RBF")
    m.X_train, m.y_train = X, y
    mean, cov = m.get_mvn_posterior(Xt, params)
    assert isinstance(mean, np.ndarray) and mean.shape == (20,) and cov.shape == (20, 20)
    mean2, cov2 = m.get_mvn_posterior(Xt, params, noiseless=True)
    np.testing.assert_array_equal(mean, mean2)
    assert not np.allclose(cov, cov2)
    mean3, cov3 = m.get_mvn_posterior(Xt, params)
    np.testing.assert_array_equal(mean, mean3)
    np.testing.assert_array_equal(cov, cov3)
    m32 = m.get_mvn_posterior(Xt.astype(np.float32), params)[0]
    assert m32.dtype == np.float32


@pytest.mark.parametrize("n", [1, 10])
@pytest.mark.parametrize("xdim", [1, 2])
def test_predict_contract(gp, n, xdim):
    """tests/test_gp.py:173-241: shapes for S=100 hand-made draws (here positive so K is SPD)"""
    X, y = dummy()
    Xt = np.linspace(1, 2, 20)
    Xt = Xt if xdim == 1 else Xt[:, None]
    rng = np.random.default_rng(0)
    samples = {"k_length": np.exp(0.3 * rng.standard_normal((100, 1))), "k_scale": np.exp(0.3 * rng.standard_normal(100)),
               "noise": np.exp(0.3 * rng.standard_normal(100))}
    m = gp.ExactGP(1, "RBF")
    m.X_train, m.y_train = X, y
    ymean, ysamp = m.predict(3, Xt, samples, n)
    assert ymean.shape == Xt.squeeze().shape and ysamp.shape == (100, n, 20)
    assert np.isfinite(ysamp).all()
    ymean2, ysamp2 = m.predict(3, Xt, samples, n)
    np.testing.assert_array_equal(ysamp, ysamp2)                      # same key -> same samples
    for bs in (2, 3, 8):
        ymb, ysb = m.predict_in_batches(3, Xt, bs, samples, n)
        assert ymb.shape == Xt.squeeze().shape and ysb.shape == (100, n, 20)
        np.testing.assert_allclose(ymb, ymean, rtol=1e-8)
    one = {k: v[0] for k, v in samples.items()}
    pm, ps = m._predict(1, Xt, one, n)
    assert pm.shape == (20,) and ps.shape == (n, 20)


def test_predict_samples_follow_the_reference_key_stream(gp):
    """ExactGP.predict(rng_key, ...) draws what the reference draws for that key: one threefry sub-key per hyper-parameter
    draw (gp.py:391), float32 normals (x64 off), y = mean + chol(cov) eps (gp.py:292) -- eps rebuilt here from the key"""
    from gpax_b200 import prng
    rng = np.random.default_rng(5)
    N, P, S, n = 200, 30, 4, 3
    X = rng.uniform(0, 1, (N, 2))
    y = np.sin(4 * X[:, 0]) + X[:, 1] + 0.1 * rng.standard_normal(N)
    Xt = rng.uniform(0, 1, (P, 2))
    samples = {"k_length": np.exp(rng.normal(np.log(0.3), 0.1, (S, 2))), "k_scale": np.exp(rng.normal(0, 0.1, S)),
               "noise": np.exp(rng.normal(np.log(0.1), 0.1, S))}
    m = gp.ExactGP(2, "RBF")
    m.X_train, m.y_train = X, y
    key = prng.PRNGKey(11)
    ymean, ysamp = m.predict(key, Xt, samples, n)
    eps = prng.mvn_eps(key, S, n, P, np.float32)
    ref_mean, _, ref_samp = oracle.predict_draws(X, y, Xt, samples, "RBF", n=n, eps=eps)
    assert_close(ymean, ref_mean, RTOL)
    assert_close(ysamp, ref_samp, 1e-6)
    _, ysamp_int = m.predict(11, Xt, samples, n)                      # an int seed is PRNGKey(seed)
    np.testing.assert_array_equal(ysamp_int, ysamp)
    one = {k: v[1] for k, v in samples.items()}
    pm, ps = m._predict(key, Xt, one, n)                              # single draw: the key itself (gp.py:292)
    e1 = prng.normal(key, (n, P), np.float32).astype(np.float64)
    rm, rc = oracle.exact_posterior(X, y, Xt, one, "RBF")
    assert_close(ps, rm[None, :] + e1 @ np.linalg.cholesky(rc).T, 1e-6)


def test_predict_negative_hyperparameters_tolerated(gp):
    """tests/test_gp.py:196-198 draws from N(0,1): about half are negative -> NaN draws, filter_nans drops them"""
    X, y = dummy()
    Xt = np.linspace(1, 2, 20)
    rng = np.random.default_rng(0)
    samples = {"k_length": rng.standard_normal((100, 1)), "k_scale": rng.standard_normal(100), "noise": rng.standard_normal(100)}
    m = gp.ExactGP(1, "RBF")
    m.X_train, m.y_train = X, y
    ymean, ysamp = m.predict(0, Xt, samples, 1)
    assert ysamp.shape == (100, 1, 20)
    _, ysf = m.predict(0, Xt, samples, 1, filter_nans=True)
    assert 0 < ysf.shape[0] < 100 and np.isfinite(ysf).all()


def test_jitter_sensitivity(gp):
    """tests/test_gp.py:353-366"""
    X, y = dummy()
    Xt = np.linspace(1, 2, 20)
    params = {"k_length": np.array([1.0]), "k_scale": 1.0, "noise": 0.1}
    m = gp.ExactGP(1, "RBF")
    m.X_train, m.y_train = X, y
    a = m.get_mvn_posterior(Xt, params, jitter=1e-6)
    b = m.get_mvn_posterior(Xt, params, jitter=1e-5)
    assert not np.array_equal(a[0], b[0]) and not np.array_equal(a[1], b[1])


def test_vigp_contract(gp):
    """tests/test_vigp.py:68-119"""
    X, y = dummy()
    params = {"k_length": np.array([1.0]), "k_scale": np.array(1.0), "noise": np.array(0.1)}
    m = gp.viGP(1, "Matern")
    m.X_train, m.y_train = X, y
    for Xt in (np.linspace(1, 2, 20), np.linspace(1, 2, 20)[:, None]):
        mean, var = m.predict(0, Xt, params)
        assert mean.shape == Xt.squeeze().shape and var.shape == Xt.squeeze().shape and (var > 0).all()
        for bs in (2, 3, 8):
            mb, vb = m.predict_in_batches(0, Xt, bs, params)
            np.testing.assert_allclose(mb, mean, rtol=1e-12)
            np.testing.assert_allclose(vb, var, rtol=1e-12)
    # var is the diagonal of get_mvn_posterior's covariance
    mean2, cov2 = m.get_mvn_posterior(np.linspace(1, 2, 20), params)
    np.testing.assert_allclose(var, np.diag(cov2), rtol=1e-10)


def test_user_kernel_callable(gp):
    """a user callable at the kernel seam (kernels.py:234-241 pass-through): Gram on the host, solve on the GPU"""
    X, y = dummy(30)
    Xt = np.linspace(1, 2, 11)
    params = {"k_length": np.array([0.7]), "k_scale": 1.0, "noise": 0.1}

    def mykernel(A, B, p, noise=0, jitter=1e-6, **kw):
        return oracle.rbf_kernel(A, B, p, noise, jitter)
    m = gp.ExactGP(1, mykernel)
    m.X_train, m.y_train = X, y
    mean, cov = m.get_mvn_posterior(Xt, params)
    rm, rc = oracle.exact_posterior(X, y, Xt, params, "RBF")
    assert_close(mean, rm, 1e-8)
    assert_close(cov, rc, 1e-8)


def test_kernel_functions_shapes(gp):
    """tests/test_kernels.py:14-40: (5,5) for scalar and ARD lengthscales, d in {1,2}"""
    rng = np.random.default_rng(0)
    for fn in (gp.RBFKernel, gp.MaternKernel, gp.PeriodicKernel):
        for d in (1, 2):
            X = rng.standard_normal((5, d))
            for ell in (np.array(1.0), np.ones(d)):
                K = fn(X, X, {"k_length": ell, "k_scale": np.array(1.0), "period": np.array(1.0)})
                assert isinstance(K, np.ndarray) and K.shape == (5, 5)


def moved(ctx, before):
    return {k: v - before[k] for k, v in ctx.path_counts().items()}


# ------------------------------------------------------------------ tall-panel factorisation (N >= 2048, int8 path on)
@pytest.mark.parametrize("ozaki", [7, -1])
@pytest.mark.parametrize("kname,N,P", [("RBF", 2500, 300), ("Matern", 3100, 129), ("Periodic", 2048, 64)])
def test_tall_panel_path_vs_oracle(gp, kname, N, P, ozaki):
    """With the int8 path on (`ozaki` 7, or -1 = planes from the conditioning bound) N >= 2048 takes potrf_tall (potrf.cuh):
    the right-hand-side rows [k_pX; y] ride under k_XX through int8 panel GEMMs with explicit inverses of the `panel`-wide
    diagonal blocks.  Ragged N (not a multiple of 512 / 128), all three kernels, mean + full covariance against the
    oracle, for every panel width and for the recursive scheme (panel = 0); the path counters prove which one ran."""
    rng = np.random.default_rng(N + P)
    d = 2
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    params = {"k_length": np.array([0.25, 0.35]), "k_scale": 1.1, "noise": 0.05, "period": 0.9}
    rmean, rcov = oracle.exact_posterior_chol(X, y, Xn, params, kname)
    K = oracle.get_kernel(kname)(X, X, params, params["noise"])
    cond = np.linalg.cond(K)
    tol = RTOL * max(1.0, cond / 1e5)
    m = gp.ExactGP(d, kname)
    m.X_train, m.y_train = X, y
    for panel in (1024, 512, 256, 0):
        with m.ctx.options(ozaki=ozaki, panel=panel):
            before = m.ctx.path_counts()
            mean, cov = m.get_mvn_posterior(Xn, params)
            c = moved(m.ctx, before)
        assert_close(mean, rmean, tol, f"mean panel={panel} ozaki={ozaki} cond={cond:.1e}")
        assert_close(cov, rcov, tol, f"cov panel={panel} ozaki={ozaki} cond={cond:.1e}")
        if panel:
            assert c["potrf_tall"] == 1 and c["panel_solve"] == -(-N // panel) and c["oz_mma"] >= c["panel_solve"], (panel, c)
        else:
            assert c["potrf_tall"] == c["panel_solve"] == 0, c
    # a failed factorisation still gives NaNs, not an exception, on this path
    bad = dict(params, k_scale=-1.0)
    with m.ctx.options(ozaki=ozaki):
        before = m.ctx.path_counts()
        mean, cov = m.get_mvn_posterior(Xn, bad)
        assert moved(m.ctx, before)["potrf_tall"] == 1
    assert np.isnan(mean).all() and np.isnan(cov).all()


@pytest.mark.parametrize("N", [300, 2500])
def test_factor_cache_reuse_with_more_and_fewer_test_points(gp, N):
    """Single-theta calls keep the factor of k_XX (the reference re-inverts it per call, gp.py:269-271).  The right-hand
    sides live under the factor in the same buffer, so a later call with MORE test points has to grow the buffer around
    the factor; at N >= 2048 with the int8 path on (set here: ozaki = 7) the reuse solves through the kept inverses of the
    diagonal blocks (trsm_tall).  Each reuse is checked against the oracle, for a handful and for many test points."""
    rng = np.random.default_rng(N)
    d = 2
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    params = {"k_length": np.array([0.3, 0.4]), "k_scale": 1.2, "noise": 0.05}
    m = gp.ExactGP(d, "Matern")
    m.X_train, m.y_train = X, y
    m.ctx.set_option("drop_factor_cache", 1)
    cond = np.linalg.cond(oracle.get_kernel("Matern")(X, X, params, params["noise"]))
    tol = RTOL * max(1.0, cond / 1e5)
    h0 = m.ctx.cache_hits()
    for k, P in enumerate((40, 10, 700, 1500, 3)):            # the first call factors, the others reuse; 700 and 1500 grow the buffer
        Xn = rng.uniform(0, 1, (P, d))
        with m.ctx.options(ozaki=7):
            before = m.ctx.path_counts()
            mean, cov = m.get_mvn_posterior(Xn, params)
            c = moved(m.ctx, before)
        rmean, rcov = oracle.exact_posterior_chol(X, y, Xn, params, "Matern")
        assert_close(mean, rmean, tol, f"mean call {k} P={P} cond={cond:.1e}")
        assert_close(cov, rcov, tol, f"cov call {k} P={P} cond={cond:.1e}")
        assert m.ctx.cache_hits() - h0 == k
        assert c["trsm_tall"] == (1 if N >= 2048 and k > 0 else 0) and c["potrf_tall"] == (1 if N >= 2048 and k == 0 else 0), (k, c)
