"""User kernel callables on the GPU: b2gp_mll_gram / b2gp_posterior_gram against an explicit-trace SciPy oracle and
against the fused entry points at the same parameters, GramLogJoint against LogJoint / NNGPLogJoint, and the models
end to end (fit, predict, predict_in_batches, acquisition functions) on callable kernels."""
import numpy as np
import pytest
import scipy.linalg as sla

import oracle
from oracle import fit_oracle as fo

pytestmark = pytest.mark.gpu

JITTER = 1e-6


@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def mll_gram_oracle(K, y, dKs):
    """log N(y; 0, (K + K^T)/2), grad_j = 1/2 sum (alpha alpha^T - K^-1) * dK_j, alpha, and the size of the terms that
    cancel in each grad_j"""
    Ks = 0.5 * (K + K.T)
    L = sla.cholesky(Ks, lower=True)
    alpha = sla.cho_solve((L, True), y)
    val = -0.5 * y @ alpha - np.log(np.diag(L)).sum() - 0.5 * len(y) * np.log(2 * np.pi)
    W = np.outer(alpha, alpha) - sla.cho_solve((L, True), np.eye(len(y)))
    grad = np.array([0.5 * np.sum(W * D) for D in dKs])
    scale = np.array([0.5 * np.sum(np.abs(W) * np.abs(D)) for D in dKs])
    return val, grad, alpha, scale


def problem(N, p, seed, noise=0.1):
    """an RBF K with noise on the diagonal and p asymmetric derivative matrices (three distinct ones cycled at large N)"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (N, 2))
    y = np.sin(4 * X[:, 0]) + 0.2 * rng.standard_normal(N)
    K = oracle.rbf_kernel(X, X, {"k_length": np.array([0.3, 0.4]), "k_scale": 1.3}, noise, JITTER)
    base = [rng.standard_normal((N, N)) for _ in range(min(p, 3 if N > 1000 else p))]
    dKs = [base[j % len(base)] * (1.0 + j) for j in range(p)]
    cond = (N * 1.3 + noise + JITTER) / (noise + JITTER)
    return K, y, dKs, cond


def counted(ctx, fn):
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


def check(ctx, K, y, dKs, cond, planes=0, device=False):
    v, g, a, sc = mll_gram_oracle(K, y, dKs)
    t = fo.tau(cond, planes)
    if device:
        args = (ctx.to_device(K), ctx.to_device(y), [ctx.to_device(D) for D in dKs])
    else:
        args = (K, y, dKs)
    (val, grad, alpha, info), c = counted(ctx, lambda: ctx.mll_gram(*args, want_grad=True, want_alpha=True))
    assert info == 0
    assert abs(val - v) <= t * abs(v), (val, v)
    assert fo.err_ratio(grad, g, sc, t) <= 1.0
    assert fo.err_ratio(alpha, a, np.abs(a).max(), t) <= 1.0
    assert c["mll_gram_trace"] == 1
    return val, grad


# ------------------------------------------------------------------ 1. b2gp_mll_gram against the oracle
@pytest.mark.parametrize("N", [1, 37, 300, 2049, 4100])
@pytest.mark.parametrize("p", [1, 4, 19])
def test_mll_gram_oracle(ctx, N, p):
    K, y, dKs, cond = problem(N, p, N + p)
    check(ctx, K, y, dKs, cond)


@pytest.mark.parametrize("N", [37, 2049])
def test_mll_gram_device_pointers(ctx, N):
    K, y, dKs, cond = problem(N, 4, 7)
    host = check(ctx, K, y, dKs, cond)
    dev = check(ctx, K, y, dKs, cond, device=True)
    assert host[0] == dev[0] and np.array_equal(host[1], dev[1])


@pytest.mark.parametrize("N", [300, 2049])
@pytest.mark.parametrize("ozaki", [7, -1])
def test_mll_gram_int8_routes(ctx, N, ozaki):
    K, y, dKs, cond = problem(N, 4, 11)
    with ctx.options(ozaki=ozaki):
        check(ctx, K, y, dKs, cond, planes=7)


def test_mll_gram_asymmetric_K_and_determinism(ctx):
    K, y, dKs, cond = problem(300, 4, 3)
    rng = np.random.default_rng(5)
    Kp = K + 1e-9 * rng.standard_normal(K.shape)          # a tiny asymmetric perturbation: the oracle factors (K + K^T)/2
    a = check(ctx, Kp, y, dKs, cond)
    b = ctx.mll_gram(Kp, y, dKs)
    assert a[0] == b[0] and np.array_equal(a[1], b[1])


def test_mll_gram_not_pd(ctx):
    K, y, dKs, _ = problem(37, 2, 1)
    K[5, 5] = -1.0
    val, grad, _, info = ctx.mll_gram(K, y, dKs)
    assert info != 0 and np.isnan(val) and np.isnan(grad).all()


def test_mll_gram_refuses_f32(ctx):
    from gpax_b200 import _ffi
    import ctypes as C
    K, y, _, _ = problem(8, 0, 1)
    v, info = C.c_double(), C.c_int()
    rc = ctx.lib.b2gp_mll_gram(ctx.h, _ffi._ptr(K), 8, 8, _ffi._ptr(y), None, 8, 0, _ffi.FLAG_F32, C.byref(v), None, None, C.byref(info))
    assert rc == -4


# ------------------------------------------------------------------ 2. cross-path against the fused likelihood
@pytest.mark.parametrize("N", [200, 2100])
def test_mll_gram_matches_fused(ctx, N):
    X, y, theta = fo.mll_problem("RBF", N, 3, N)
    d = 3
    ell, scale, noise = theta[:d], theta[d], theta[d + 1]
    K0 = ctx.gram("RBF", X, X, ell, scale, 1.0, 0.0, True)
    K = K0 + (noise + JITTER) * np.eye(N)
    dKs = [K0 * (X[:, k][:, None] - X[:, k][None, :]) ** 2 / ell[k] ** 2 for k in range(d)] + [K0, noise * np.eye(N)]
    val, grad, _, info = ctx.mll_gram(K, y, dKs)
    v, g, _, info2 = ctx.mll("RBF", X, y, theta, JITTER, want_grad=True)
    assert info == 0 and info2 == 0
    np.testing.assert_allclose(val, v, rtol=1e-10)
    np.testing.assert_allclose(grad, g[:d + 2], rtol=1e-9, atol=1e-9 * np.abs(g).max())


# ------------------------------------------------------------------ 3. GramLogJoint against the fused log joints
def rbf_callable(X, Z, params, noise=0, jitter=1e-6, **kw):
    return oracle.rbf_kernel(X, Z, params, noise, jitter)


def _model_xy(N, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (N, d))
    return X, np.sin(4 * X[:, 0]) + 0.1 * rng.standard_normal(N)


def test_gram_log_joint_matches_log_joint(ctx):
    import gpax_b200 as gp
    from gpax_b200.inference import GramLogJoint, LogJoint, make_log_joint
    X, y = _model_xy(120, 2, 0)
    mc, mf = gp.ExactGP(2, rbf_callable, ctx=ctx), gp.ExactGP(2, "RBF", ctx=ctx)
    for m in (mc, mf):
        m.X_train, m.y_train = X, y
    lc, lf = make_log_joint(mc), LogJoint(mf)
    assert isinstance(lc, GramLogJoint) and lc.dim == lf.dim
    rng = np.random.default_rng(1)
    for _ in range(5):
        u = lf.init_u() + 0.3 * rng.standard_normal(lf.dim)
        for jac in (True, False):
            vc, gc = lc(u, jac)
            vf, gf = lf(u, jac)
            np.testing.assert_allclose(vc, vf, rtol=1e-10)
            np.testing.assert_allclose(gc, gf, rtol=1e-6, atol=1e-6 * np.abs(gf).max())


def test_gram_log_joint_nngp(ctx):
    import gpax_b200 as gp
    from gpax_b200 import priors as P
    from gpax_b200.inference import NNGPLogJoint, make_log_joint

    def nngp_prior():
        return {"var_b": P.sample("var_b", P.LogNormal(0.0, 1.0)), "var_w": P.sample("var_w", P.LogNormal(0.0, 1.0))}
    X, y = _model_xy(90, 2, 2)
    from gpax_b200.kernels import NNGPKernel
    mc = gp.ExactGP(2, NNGPKernel("erf", 3), kernel_prior=nngp_prior, ctx=ctx)
    mf = gp.iBNN(2, depth=3, activation="erf", ctx=ctx)
    for m in (mc, mf):
        m.X_train, m.y_train = X, y
    lc, lf = make_log_joint(mc), NNGPLogJoint(mf)
    rng = np.random.default_rng(3)
    for _ in range(5):
        u = lf.init_u() + 0.3 * rng.standard_normal(3)
        vc, gc = lc(u, True)
        vf, gf = lf(u, True)
        np.testing.assert_allclose(vc, vf, rtol=1e-10)
        np.testing.assert_allclose(gc, gf, rtol=1e-6, atol=1e-6 * np.abs(gf).max())


def test_gram_log_joint_program_with_mean(ctx):
    """an extra kernel site and a probabilistic mean function against ProgramLogJoint on the fused RBF"""
    import gpax_b200 as gp
    from gpax_b200 import priors as P
    from gpax_b200.inference import ProgramLogJoint, make_log_joint

    def kprior():
        a = P.sample("a", P.LogNormal(0.0, 1.0))
        return {"k_length": P.sample("k_length", P.LogNormal(0.0, 1.0)), "k_scale": a * P.sample("k_s", P.LogNormal(0.0, 1.0))}

    def mean_fn(X, p):
        return p["m0"] + p["m1"] * X[:, 0]

    def mprior():
        return {"m0": P.sample("m0", P.Normal(0.0, 1.0)), "m1": P.sample("m1", P.Normal(0.0, 1.0))}
    X, y = _model_xy(80, 1, 4)
    kw = dict(mean_fn=mean_fn, kernel_prior=kprior, mean_fn_prior=mprior, ctx=ctx)
    mc, mf = gp.ExactGP(1, rbf_callable, **kw), gp.ExactGP(1, "RBF", **kw)
    for m in (mc, mf):
        m.X_train, m.y_train = X, y
    lc, lf = make_log_joint(mc), ProgramLogJoint(mf)
    assert [s.name for s in lc.sites] == [s.name for s in lf.sites]
    rng = np.random.default_rng(5)
    for _ in range(5):
        u = lf.init_u() + 0.3 * rng.standard_normal(lf.dim)
        vc, gc = lc(u, True)
        vf, gf = lf(u, True)
        np.testing.assert_allclose(vc, vf, rtol=1e-10)
        np.testing.assert_allclose(gc, gf, rtol=1e-6, atol=1e-6 * np.abs(gf).max())


# ------------------------------------------------------------------ 4. posterior_gram against b2gp_posterior
@pytest.mark.parametrize("kind", ["RBF", "Periodic", "Matern"])
@pytest.mark.parametrize("N,P", [(40, 1), (40, 33), (2100, 33)])
def test_posterior_gram_matches_fused(ctx, kind, N, P):
    rng = np.random.default_rng(N + P)
    S, d, n = 5, 2, 3
    X, Xn = rng.uniform(0, 1, (N, d)), rng.uniform(0, 1, (P, d))
    y = np.sin(4 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    theta = np.column_stack([rng.uniform(0.3, 0.6, (S, d)), rng.uniform(0.8, 1.5, S), rng.uniform(0.05, 0.2, S),
                             rng.uniform(0.7, 1.2, S)])
    eps = rng.standard_normal((S, n, P))
    Kxx, Kpx, Kpp = [], [], []
    for th in theta:
        ell, sc, nz, per = th[:d], th[d], th[d + 1], th[d + 2]
        Kxx.append(ctx.gram(kind, X, X, ell, sc, per, nz + JITTER, True))
        Kpx.append(ctx.gram(kind, Xn, X, ell, sc, per, 0.0, False))
        Kpp.append(ctx.gram(kind, Xn, Xn, ell, sc, per, nz + JITTER, True))
    Kxx, Kpx, Kpp = np.stack(Kxx), np.stack(Kpx), np.stack(Kpp)
    want = ("mean", "var", "cov")
    got = ctx.posterior_gram(Kxx, Kpx, Kpp, y, want, eps)
    ref = ctx.posterior(kind, X, y, Xn, theta, False, JITTER, want, eps)
    rtol = 1e-9 if kind == "Matern" else 1e-12
    for k in ("mean", "var", "cov", "y_sampled"):
        np.testing.assert_allclose(got[k], ref[k], rtol=rtol, atol=rtol * np.abs(ref[k]).max(), err_msg=k)
    diag = ctx.posterior_gram(Kxx, Kpx, np.diagonal(Kpp, axis1=1, axis2=2), y, ("mean", "var"), kpp_diag=True)
    np.testing.assert_array_equal(diag["var"], got["var"])
    np.testing.assert_array_equal(diag["mean"], got["mean"])


# ------------------------------------------------------------------ 5. end to end
@pytest.mark.parametrize("noiseless", [False, True])
def test_predict_callable_matches_builtin(ctx, noiseless):
    import gpax_b200 as gp
    X, y = _model_xy(60, 1, 6)
    Xt = np.linspace(0, 1, 25)
    rng = np.random.default_rng(7)
    samples = {"k_length": rng.uniform(0.3, 0.6, (6, 1)), "k_scale": rng.uniform(0.8, 1.5, 6), "noise": rng.uniform(0.05, 0.2, 6)}
    mc, mf = gp.ExactGP(1, rbf_callable, ctx=ctx), gp.ExactGP(1, "RBF", ctx=ctx)
    for m in (mc, mf):
        m.X_train, m.y_train = X, y
    a = mc.predict(0, Xt, samples, n=2, noiseless=noiseless)
    b = mf.predict(0, Xt, samples, n=2, noiseless=noiseless)
    for u, v in zip(a, b):
        np.testing.assert_allclose(u, v, rtol=1e-9, atol=1e-9 * np.abs(v).max())
    a = mc.predict_in_batches(0, Xt, 10, samples, n=2, noiseless=noiseless)
    b = mf.predict_in_batches(0, Xt, 10, samples, n=2, noiseless=noiseless)
    for u, v in zip(a, b):
        np.testing.assert_allclose(u, v, rtol=1e-9, atol=1e-9 * np.abs(v).max())


def test_fit_callable_sites(ctx):
    import gpax_b200 as gp
    X, y = _model_xy(40, 2, 8)
    m = gp.ExactGP(2, rbf_callable, ctx=ctx)
    m.fit(0, X, y, num_warmup=100, num_samples=100, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert set(s) == {"k_length", "k_scale", "noise"}
    assert s["k_length"].shape == (100, 2) and s["k_scale"].shape == (100,) and s["noise"].shape == (100,)
    assert all(np.isfinite(v).all() for v in s.values())


def test_vigp_callable_map_matches_builtin(ctx):
    import gpax_b200 as gp
    X, y = _model_xy(50, 1, 9)
    mc, mf = gp.viGP(1, rbf_callable, ctx=ctx), gp.viGP(1, "RBF", ctx=ctx)
    for m in (mc, mf):
        m.fit(0, X, y, num_steps=500, step_size=5e-3, progress_bar=False, print_summary=False)
    for k in ("k_length", "k_scale", "noise"):
        np.testing.assert_allclose(mc.get_samples()[k], mf.get_samples()[k], rtol=1e-5)


def test_set_kernel_fn_linear_plus_rbf(ctx):
    import gpax_b200 as gp
    from gpax_b200.acquisition import EI, optimize_acq
    from gpax_b200.utils import set_kernel_fn
    from gpax_b200 import priors as P
    kern = set_kernel_fn(_lin_rbf)

    def kprior():
        return {"k_length": P.sample("k_length", P.LogNormal(0.0, 1.0)), "k_scale": P.sample("k_scale", P.LogNormal(0.0, 1.0)),
                "k_lin": P.sample("k_lin", P.LogNormal(0.0, 1.0))}
    X, y = _model_xy(30, 1, 10)
    m = gp.ExactGP(1, kern, kernel_prior=kprior, ctx=ctx)
    m.fit(1, X, y, num_warmup=50, num_samples=20, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert set(s) == {"k_length", "k_scale", "k_lin", "noise"} and s["k_lin"].shape == (20,)
    Xt = np.linspace(-0.2, 1.2, 17)
    rng = np.random.default_rng(0)
    mean, ys = m.predict(rng, Xt, s, n=2)
    assert mean.shape == (17,) and ys.shape == (20, 2, 17)
    # mean at the drawn parameters against a NumPy posterior
    out = m._posterior_batched(Xt, s, True, False, ("mean",))
    for i in range(20):
        p = {k: v[i] for k, v in s.items()}
        Kxx = kern(X, X, p, p["noise"])
        Kpx = kern(Xt[:, None], X, p, jitter=0.0)
        ref = Kpx @ np.linalg.solve(Kxx, y)
        np.testing.assert_allclose(out["mean"][i], ref, rtol=1e-8, atol=1e-8 * np.abs(ref).max())
    ei = EI(0, m, Xt, maximize=True)
    assert ei.shape == (17,) and np.isfinite(ei).all()
    x = optimize_acq(0, m, EI, num_initial_guesses=3, lower_bound=0.0, upper_bound=1.0, maximize=True)
    assert np.all(np.isfinite(np.asarray(x)))


def _lin_rbf(X, Z, k_lin, k_length, k_scale):
    d2 = ((X[:, None, :] - Z[None, :, :]) / k_length) ** 2
    return k_lin * X @ Z.T + k_scale * np.exp(-0.5 * d2.sum(-1))
