"""GPU: b2gp_mll_draws_v, S noise-vector likelihoods in lock-step, and the MeasuredNoiseGP / VarNoiseGP fits with prior
programs and noise mean functions whose chains run on it under chain_method="vectorized".

Draw s of ctx.mll_draws_v must be ctx.mll(theta[s], yres[s], noise_vec=noise_vec[s]) bit for bit on every route and
however the draws are grouped: that is what keeps vectorized chains identical to sequential ones."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_hsk.npz")


@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def inputs(kind, N, S, d=2, seed=0):
    rng = np.random.default_rng(seed + 7 * N + S)
    X = rng.uniform(0, 1, (N, d))
    Y = np.sin(5 * X[:, 0])[None] * np.cos(3 * X[:, 1])[None] + 0.1 * rng.standard_normal((S, N))
    NV = np.exp(rng.normal(-3.0, 0.5, (S, N)))
    if kind.startswith("NNGP"):     # (depth, unused, var_w, noise, var_b)
        theta = np.column_stack([np.full(S, 2.0), np.zeros((S, d - 1)), rng.uniform(0.8, 1.5, S), rng.uniform(0.02, 0.1, S),
                                 rng.uniform(0.05, 0.3, S)])
    else:
        theta = np.column_stack([rng.uniform(0.2, 0.5, (S, d)), rng.uniform(0.7, 1.3, S), rng.uniform(0.0, 0.05, S),
                                 rng.uniform(0.6, 1.2, S)])
    return X, Y, NV, theta


def same(a, b):
    return np.shape(a) == np.shape(b) and np.array_equal(a, b, equal_nan=True)


def check_bits(ctx, kind, X, Y, NV, theta, shared_y, shared_nv):
    """mll_draws_v against one ctx.mll(noise_vec=...) per draw: value, gradient, alpha, grad_noise_vec and info"""
    val, grad, alpha, gnv, info = ctx.mll_draws_v(kind, X, Y[0] if shared_y else Y, theta, NV[0] if shared_nv else NV,
                                                  want_grad=True, want_alpha=True)
    for s in range(theta.shape[0]):
        v, g, a, i, gn = ctx.mll(kind, X, Y[0] if shared_y else Y[s], theta[s], want_grad=True, want_alpha=True,
                                 noise_vec=NV[0] if shared_nv else NV[s])
        assert info[s] == i
        assert same(np.array(val[s]), np.array(v)), (s, val[s], v)
        assert same(grad[s], g) and same(gnv[s], gn), s
        if i == 0:
            assert same(alpha[s], a), s
    return val, grad, alpha, gnv, info


def counted(ctx, fn):
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic", "NNGP_erf"])
@pytest.mark.parametrize("N", [1, 17, 129, 700])
def test_draws_v_match_mll_v_bit_for_bit(ctx, kind, N):
    for S in (1, 3, 8):
        X, Y, NV, theta = inputs(kind, N, S)
        for shared_y, shared_nv in ((True, True), (False, False), (True, False), (False, True)):
            info = check_bits(ctx, kind, X, Y, NV, theta, shared_y, shared_nv)[4]
            assert (info == 0).all()


@pytest.mark.parametrize("kind", ["RBF", "Periodic", "NNGP_erf"])
def test_tall_fp64_route(ctx, kind):
    X, Y, NV, theta = inputs(kind, 700, 3)
    with ctx.options(tall_min_fp64=256, panel=256):
        _, moved = counted(ctx, lambda: check_bits(ctx, kind, X, Y, NV, theta, False, False))
    assert moved["potrf_tall_fp64"] == 6 and moved["mll_draws_batch"] == 1


@pytest.mark.parametrize("kind", ["RBF", "NNGP_erf"])
def test_int8_route_runs_per_draw(ctx, kind):
    X, Y, NV, theta = inputs(kind, 700, 3)
    with ctx.options(ozaki=7, tall_min=512):
        _, moved = counted(ctx, lambda: check_bits(ctx, kind, X, Y, NV, theta, True, False))
    assert moved["mll_draws_batch"] == 3 and moved["potrf_tall"] == 6


def test_group_split_keeps_the_bits(ctx):
    X, Y, NV, theta = inputs("Matern", 300, 8)
    ref = ctx.mll_draws_v("Matern", X, Y, theta, NV, want_alpha=True)
    for B, groups in ((1, 8), (3, 3), (8, 1)):
        with ctx.options(draw_batch=B):
            got, moved = counted(ctx, lambda: check_bits(ctx, "Matern", X, Y, NV, theta, False, False))
        assert moved["mll_draws_batch"] == groups
        for a, b in zip(got, ref):
            assert same(a, b)


def test_launches_do_not_grow_with_draws(ctx):
    X, Y, NV, theta = inputs("RBF", 129, 8)
    ctx.mll_draws_v("RBF", X, Y[0], theta[:1], NV[0])
    one = ctx.last_timing()["launches"]
    _, moved = counted(ctx, lambda: ctx.mll_draws_v("RBF", X, Y[0], theta, NV))
    assert ctx.last_timing()["launches"] == one and moved["mll_draws_batch"] == 1
    # the noise-vector form adds the diagonal, d value / d noise_vec and its copy out to b2gp_mll_draws' sequence
    ctx.mll_draws("RBF", X, Y[0], theta[:1])
    assert one == ctx.last_timing()["launches"] + 3


def test_failed_draw_is_isolated(ctx):
    X, Y, NV, theta = inputs("RBF", 129, 4)
    NV[2, 5] = -5.0                                       # K + diag(noise_vec) is not positive definite
    val, grad, alpha, gnv, info = check_bits(ctx, "RBF", X, Y, NV, theta, False, False)
    assert info[2] != 0 and np.isnan(val[2]) and np.isnan(grad[2]).all() and np.isnan(alpha[2]).all() and np.isnan(gnv[2]).all()
    assert (info[[0, 1, 3]] == 0).all() and np.isfinite(val[[0, 1, 3]]).all() and np.isfinite(gnv[[0, 1, 3]]).all()


def test_refusals_before_any_launch(ctx):
    from gpax_b200 import _ffi
    X, Y, NV, theta = inputs("RBF", 64, 2)
    val, info = np.zeros(2), np.zeros(2, dtype=np.int32)
    p = lambda a: C.c_void_p(a.ctypes.data)     # noqa: E731
    for flags in (_ffi.FLAG_F32, _ffi.FLAG_DEVICE_PTRS):
        before = ctx.path_counts()
        rc = ctx.lib.b2gp_mll_draws_v(ctx.h, _ffi.KERNEL_RBF, p(X), 64, p(Y), 64, 2, 2, p(theta), p(NV), 64, 1e-6, flags, p(val),
                                      None, None, None, p(info))
        assert rc == -4 and ctx.path_counts() == before
    before = ctx.path_counts()
    gnv = np.zeros((2, 64))                                # grad_noise_vec without grad
    assert ctx.lib.b2gp_mll_draws_v(ctx.h, _ffi.KERNEL_RBF, p(X), 64, p(Y), 64, 2, 2, p(theta), p(NV), 64, 1e-6, 0, p(val), None,
                                    None, p(gnv), p(info)) != 0
    assert ctx.lib.b2gp_mll_draws_v(ctx.h, _ffi.KERNEL_RBF, p(X), 64, p(Y), 64, 2, 2, p(theta), None, 0, 1e-6, 0, p(val), None,
                                    None, None, p(info)) != 0
    assert ctx.path_counts() == before
    with pytest.raises(ValueError):
        ctx.mll_draws_v("RBF", X, Y, theta, NV[:, :10])
    with pytest.raises(_ffi.B200GPError):                  # NNGP depth checked per draw, before any launch
        bad = inputs("NNGP_erf", 64, 2)[3]
        bad[1, 0] = 1.5
        ctx.mll_draws_v("NNGP_erf", X, Y[0], bad, NV[0])
    assert ctx.path_counts() == before


# ---------------------------------------------------------------------------------------------- fits
def noise_fn(x, params):                                  # the reference's tests/test_hskgp.py
    return params["a"] + params["b"] * x


def noise_fn_prior():
    from gpax_b200 import priors as numpyro
    return {"a": numpyro.sample("a", numpyro.distributions.Normal(0, 1)),
            "b": numpyro.sample("b", numpyro.distributions.Normal(0, 1))}


def noise_kernel_prior():
    from gpax_b200 import priors as numpyro
    return {"k_noise_length": numpyro.sample("k_noise_length", numpyro.distributions.LogNormal(0.0, 0.5)),
            "k_noise_scale": numpyro.sample("k_noise_scale", numpyro.distributions.Gamma(2.0, 2.0))}


def kernel_prior():
    from gpax_b200 import priors as numpyro
    return {"k_length": numpyro.sample("k_length", numpyro.distributions.Gamma(2.0, 2.0)),
            "k_scale": numpyro.sample("k_scale", numpyro.distributions.LogNormal(0.0, 1.0))}


def mean_fn(x, params):
    return params["c"] * x ** 2


def mean_fn_prior():
    from gpax_b200 import priors as numpyro
    return {"c": numpyro.sample("c", numpyro.distributions.LogNormal(2.0, 0.5))}


def _dummy(n=8, seed=0):                                  # get_dummy_data of the reference's tests
    rng = np.random.default_rng(seed)
    X = np.linspace(1, 2, n) + 0.1 * rng.standard_normal(n)
    return X, 10 * X ** 2


FITS = {
    "VarNoiseGP": (lambda c: __import__("gpax_b200").VarNoiseGP(1, "RBF", ctx=c), False),
    "noise_mean_fn": (lambda c: __import__("gpax_b200").VarNoiseGP(1, "RBF", noise_mean_fn=noise_fn,
                                                                    noise_mean_fn_prior=noise_fn_prior, ctx=c), False),
    "noise_and_regular_mean_fn": (lambda c: __import__("gpax_b200").VarNoiseGP(1, "RBF", mean_fn=lambda x: 8 * x ** 2,
                                                                                noise_mean_fn=noise_fn,
                                                                                noise_mean_fn_prior=noise_fn_prior, ctx=c), False),
    "noise_kernel_prior": (lambda c: __import__("gpax_b200").VarNoiseGP(1, "RBF", noise_kernel_prior=noise_kernel_prior, ctx=c),
                           False),
    "MeasuredNoiseGP_programs": (lambda c: __import__("gpax_b200").MeasuredNoiseGP(1, "RBF", kernel_prior=kernel_prior,
                                                                                   mean_fn=mean_fn, mean_fn_prior=mean_fn_prior,
                                                                                   ctx=c), True),
}


@pytest.mark.filterwarnings("ignore::UserWarning")
@pytest.mark.parametrize("name", list(FITS))
def test_vectorized_fit_matches_sequential(ctx, name):
    make, measured = FITS[name]
    runs = {}
    for method in ("sequential", "vectorized"):
        m = make(ctx)
        X, y = _dummy()
        args = (X, y, np.full(X.size, 0.05)) if measured else (X, y)
        calls = {"mll": 0, "mll_draws": 0, "mll_draws_v": 0}
        for k in calls:
            def wrap(*a, _f=getattr(ctx, k), _k=k, **kw):
                calls[_k] += 1
                return _f(*a, **kw)
            setattr(ctx, k, wrap)
        try:
            m.fit(0, *args, num_warmup=10, num_samples=10, num_chains=3, chain_method=method, progress_bar=False,
                  print_summary=False)
        finally:
            for k in calls:
                delattr(ctx, k)
        runs[method] = (m.mcmc.get_samples(group_by_chain=True), m.mcmc.stats, calls)
    (s_seq, st_seq, c_seq), (s_vec, st_vec, c_vec) = runs["sequential"], runs["vectorized"]
    assert list(s_seq) == list(s_vec)
    for k in s_seq:
        assert np.asarray(s_seq[k]).shape[:2] == (3, 10) and same(np.asarray(s_seq[k]), np.asarray(s_vec[k])), k
    assert st_seq == st_vec
    rounds = max(np.diff([0] + [s["grad_evals"] for s in st_vec]))
    assert c_vec["mll_draws_v"] == rounds and c_vec["mll"] == 0
    assert c_vec["mll_draws"] == (0 if measured else rounds)
    assert c_seq["mll_draws"] == 0 and c_seq["mll_draws_v"] == 0


def test_noise_mean_fit_recovers_a_growing_noise(ctx):
    """the trend data of test_gpu_f_rows.test_variant_fits_run, with noise_mean_fn = a + b x under a prior"""
    import gpax_b200
    rng = np.random.default_rng(4)
    X = np.sort(rng.uniform(0, 1, 60))[:, None]
    noise_sd = 0.05 + 0.25 * X[:, 0]
    y = np.sin(6 * X[:, 0]) + noise_sd * rng.standard_normal(60)
    m = gpax_b200.VarNoiseGP(1, "RBF", noise_mean_fn=noise_fn, noise_mean_fn_prior=noise_fn_prior, ctx=ctx)
    m.fit(1, X, y, num_warmup=60, num_samples=30, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert s["log_var"].shape == (30, 60) and s["a"].shape == (30,)
    dv = m.get_data_var_samples()
    assert dv.shape == (30, 60) and np.isfinite(dv).all()
    assert np.median(dv[:, 45:]) > np.median(dv[:, :15])            # the inferred noise grows with x, as the data's does
    mean, ys = m.predict(1, np.array([[0.1], [0.9]]), n=1)
    assert np.isfinite(mean).all() and np.isfinite(ys).all()


@pytest.mark.parametrize("tag", ["fixed", "prior"])
def test_posterior_matches_the_reference(ctx, tag):
    import gpax_b200
    g = np.load(GOLDEN)

    def noise_fixed(x):
        return 0.02 + 0.1 * x

    p = {k[2:]: g[k] for k in g.files if k.startswith("p_")}
    kw = dict(noise_mean_fn=noise_fixed) if tag == "fixed" else dict(noise_mean_fn=noise_fn, noise_mean_fn_prior=noise_fn_prior)
    m = gpax_b200.VarNoiseGP(1, "RBF", noise_kernel="RBF", mean_fn=lambda x, q: q["c"] * x ** 2, mean_fn_prior=mean_fn_prior,
                             ctx=ctx, **kw)
    m.X_train, m.y_train = g["Xtr"], g["ytr"]
    params = dict(p, log_var=g["log_var"], noise=0.0)
    mean, cov = m.get_mvn_posterior(g["Xte"], params)
    # the reference inverts k_XX explicitly: entries far below the diagonal's scale carry its rounding, hence the atol
    tol = dict(rtol=1e-6, atol=1e-6 * np.abs(g[f"{tag}_cov"]).max())
    np.testing.assert_allclose(mean, g[f"{tag}_mean"], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(cov, g[f"{tag}_cov"], **tol)
    # the batched path (predict) evaluates the noise mean per draw: two draws at the same parameters give the same moments
    S2 = {k: np.stack([np.asarray(v)] * 2) for k, v in params.items()}
    out, pv = m._both_posteriors(g["Xte"], S2, True, ("mean", "cov"))
    for s in range(2):
        c = out["cov"][s].copy()
        c[np.diag_indices_from(c)] += pv[s]
        np.testing.assert_allclose(out["mean"][s], g[f"{tag}_mean"], rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(c, g[f"{tag}_cov"], **tol)
