"""GPU: viSparseGP with a user kernel callable -- b2gp_sparse_elbo_gram and b2gp_sparse_posterior_gram against the
NumPy oracle (tests/sparse_gram_oracle.py), against the fused entry points on callables equal to the built-in kernels,
and the model end to end (fit, predict, mean functions, acquisitions)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle  # noqa: E402
from oracle import fit_oracle as fo  # noqa: E402
import sparse_gram_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_vectors_sparse_callable.npz")


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    return _ffi.default_context()


def _problem(M, N, d, seed, grid=False):
    """RBF blocks on well-separated inducing points (cond(Kuu) stays small), random asymmetric directions"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (N, d))
    if grid:
        g = int(round(M ** (1 / d)))
        Xu = np.stack(np.meshgrid(*[np.linspace(0, 1, g)] * d), -1).reshape(-1, d)
        ell = 0.6 / g
    else:
        Xu = np.sort(rng.uniform(0, 1, (M, d)), axis=0) if M > 1 else rng.uniform(0, 1, (1, d))
        Xu[:, 0] = np.linspace(0, 1, M) if M > 1 else Xu[:, 0]
        ell = 0.5 / M
    p = {"k_length": np.full(d, ell), "k_scale": 1.3}
    Kuu = oracle.rbf_kernel(Xu, Xu, p, jitter=1e-6)
    Kuf = oracle.rbf_kernel(Xu, X, p, jitter=0)
    kff = np.full(N, 1.3)
    y = np.sin(5 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    return Kuu, Kuf, kff, y, rng


def _dirs(rng, M, N, p, q, nulls=False):
    dirs = [(rng.standard_normal((M, M)), rng.standard_normal((M, N)), rng.standard_normal(N)) for _ in range(p)]
    rdirs = [(rng.standard_normal((M, M)), rng.standard_normal((M, N))) for _ in range(q)]
    if nulls and p >= 3:
        dirs[0] = (None, dirs[0][1], dirs[0][2])
        dirs[1] = (dirs[1][0], None, None)
        dirs[2] = (None, None, None)
    if nulls and q >= 2:
        rdirs[1] = (None, rdirs[1][1])
    return dirs, rdirs


def _check(r, ref):
    v, g, gln, rows, alpha = ref
    assert r["info"] == 0
    np.testing.assert_allclose(r["value"], v, rtol=1e-10)
    for got, want in ((r["grad"], g), (r["grad_rows"], rows), (r["alpha"], alpha), (r["grad_log_noise"], gln)):
        want = np.asarray(want)
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-9 * max(1.0, float(np.abs(want).max(initial=0.0))))


@pytest.mark.parametrize("M,N,d,p,q,nulls,grid", [
    (1, 45, 1, 2, 1, False, False),
    (7, 301, 2, 3, 2, True, False),
    (256, 1000, 2, 2, 2, False, True),
    (40, 40, 1, 1, 1, False, False),       # M == N
    (7, 77, 2, 0, 2, False, False),        # p = 0
    (7, 77, 2, 3, 0, True, False),         # q = 0
])
def test_elbo_gram_matches_oracle(ctx, M, N, d, p, q, nulls, grid):
    Kuu, Kuf, kff, y, rng = _problem(M, N, d, M + N, grid)
    dirs, rdirs = _dirs(rng, M, N, p, q, nulls)
    ref = so.elbo_gram_grad(Kuu, Kuf, kff, y, 0.05, dirs, rdirs)
    _check(ctx.sparse_elbo_gram(Kuu, Kuf, kff, y, 0.05, dirs, rdirs, want_alpha=True), ref)


def test_elbo_gram_device_pointers_and_determinism(ctx):
    M, N = 7, 301
    Kuu, Kuf, kff, y, rng = _problem(M, N, 2, 9)
    dirs, rdirs = _dirs(rng, M, N, 3, 2, nulls=True)
    ref = so.elbo_gram_grad(Kuu, Kuf, kff, y, 0.05, dirs, rdirs)
    host = [ctx.sparse_elbo_gram(Kuu, Kuf, kff, y, 0.05, dirs, rdirs, want_alpha=True) for _ in range(2)]
    for k in ("grad", "grad_rows", "alpha"):
        assert np.array_equal(host[0][k], host[1][k])
    assert host[0]["value"] == host[1]["value"] and host[0]["grad_log_noise"] == host[1]["grad_log_noise"]
    dv = lambda a: None if a is None else ctx.to_device(np.ascontiguousarray(a))   # noqa: E731
    r = ctx.sparse_elbo_gram(dv(Kuu), dv(Kuf), dv(kff), dv(y), 0.05, [tuple(dv(b) for b in t) for t in dirs],
                             [tuple(dv(b) for b in t) for t in rdirs], want_alpha=True)
    _check(r, ref)


def test_elbo_gram_failures_and_refusals(ctx):
    from gpax_b200 import _ffi
    M, N = 7, 50
    Kuu, Kuf, kff, y, rng = _problem(M, N, 1, 4)
    dirs, rdirs = _dirs(rng, M, N, 2, 1)
    bad = Kuu.copy()
    bad[3, 3] = -1.0
    r = ctx.sparse_elbo_gram(bad, Kuf, kff, y, 0.05, dirs, rdirs, want_alpha=True)
    assert r["info"] > 0 and np.isnan(r["value"]) and np.isnan(r["grad"]).all() and np.isnan(r["grad_rows"]).all()
    assert np.isnan(r["alpha"]).all() and np.isnan(r["grad_log_noise"])
    _check(ctx.sparse_elbo_gram(Kuu, Kuf, kff, y, 0.05, dirs, rdirs, want_alpha=True),
           so.elbo_gram_grad(Kuu, Kuf, kff, y, 0.05, dirs, rdirs))
    # a negative noise makes I + W W^T / noise indefinite: the inner factorisation fails
    r = ctx.sparse_elbo_gram(Kuu, 30 * Kuf, kff, y, -0.05, dirs, rdirs)
    assert r["info"] < 0 and np.isnan(r["value"]) and np.isnan(r["grad"]).all()
    with pytest.raises(_ffi.B200GPError):
        ctx.sparse_elbo_gram(Kuu, Kuf, kff, y, 0.05, dirs, rdirs, flags=_ffi.FLAG_F32)
    with pytest.raises(_ffi.B200GPError):
        ctx.sparse_posterior_gram(Kuu, Kuf, y, 0.05, Kuf[:, :5], np.ones(5), want=("mean", "cov"), kss_diag=True)


def test_path_counter(ctx):
    Kuu, Kuf, kff, y, rng = _problem(7, 60, 1, 2)
    before = ctx.path_counts()["sparse_gram_trace"]
    ctx.sparse_elbo_gram(Kuu, Kuf, kff, y, 0.05, *_dirs(rng, 7, 60, 2, 1))
    assert ctx.path_counts()["sparse_gram_trace"] == before + 1


def test_sparse_elbo_alpha_keeps_the_other_outputs(ctx):
    Xu, X, y, theta = fo.elbo_problem("Matern", 30, 500, 2, seed=11)
    a = ctx.sparse_elbo("Matern", Xu, X, y, theta)
    b = ctx.sparse_elbo("Matern", Xu, X, y, theta, want_alpha=True)
    assert a[0] == b[0] and a[3] == b[3] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    blocks = (oracle.matern_kernel(Xu, Xu, _params(theta, 2), jitter=1e-6), oracle.matern_kernel(Xu, X, _params(theta, 2), jitter=0),
              np.diag(oracle.matern_kernel(X, X, _params(theta, 2), jitter=0)))
    np.testing.assert_allclose(b[4], so.elbo_gram_grad(*blocks, y, theta[3])[4], rtol=1e-8, atol=1e-8)


def _params(theta, d):
    return {"k_length": theta[:d], "k_scale": float(theta[d]), "period": float(theta[d + 2])}


KERNELS = {"RBF": oracle.rbf_kernel, "Matern": oracle.matern_kernel, "Periodic": oracle.periodic_kernel}


@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
def test_callables_equal_to_builtins_give_the_fused_bound(ctx, kind):
    from gpax_b200 import inference
    from gpax_b200.sparse_gp import viSparseGP
    d = 2
    Xu, X, y, theta = fo.elbo_problem(kind, 12, 400, d, seed=9)   # cond(Kuu) ~ 1e4: differenced blocks lose ~cond * 1e-11
    v0, g0, gx0, info0 = ctx.sparse_elbo(kind, Xu, X, y, theta, 1e-6)
    m = viSparseGP(d, KERNELS[kind], ctx=ctx)
    m.X_train, m.y_train = X, y
    lj = inference.SparseGramLogJoint(m, Xu, jitter=1e-6)
    kp = _params(theta, d)
    blocks = lj._blocks(kp)
    h = 1e-5
    names = [("k_length", k) for k in range(d)] + [("k_scale", None)] + ([("period", None)] if kind == "Periodic" else [])
    dirs = []
    for name, k in names:   # d / dlog(theta) by central differences of the callable
        kpp, kpm = dict(kp), dict(kp)
        if k is None:
            kpp[name], kpm[name] = kp[name] * np.exp(h), kp[name] * np.exp(-h)
        else:
            kpp[name], kpm[name] = kp[name].copy(), kp[name].copy()
            kpp[name][k] *= np.exp(h)
            kpm[name][k] *= np.exp(-h)
        dirs.append(tuple((a - b) / (2 * h) for a, b in zip(lj._blocks(kpp), lj._blocks(kpm))))
    r = ctx.sparse_elbo_gram(*blocks, y, theta[d + 1], dirs, lj._xu_dirs(kp))
    assert r["info"] == 0 == info0
    np.testing.assert_allclose(r["value"], v0, rtol=1e-10)
    want = np.concatenate([g0[:d + 1], g0[d + 2:] if kind == "Periodic" else []])
    np.testing.assert_allclose(r["grad"], want, rtol=1e-6, atol=1e-6 * np.abs(want).max())
    np.testing.assert_allclose(r["grad_log_noise"], g0[d + 1], rtol=1e-9)
    np.testing.assert_allclose(r["grad_rows"].T, gx0, rtol=1e-6, atol=1e-6 * np.abs(gx0).max())


@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
@pytest.mark.parametrize("noiseless", [False, True])
def test_posterior_gram_matches_the_fused_posterior(ctx, kind, noiseless):
    d = 2
    Xu, X, y, theta = fo.elbo_problem(kind, 40, 600, d, seed=13)
    Xs = np.random.default_rng(1).uniform(0, 1, (77, d))
    kp, noise = _params(theta, d), theta[d + 1]
    k = KERNELS[kind]
    ref = ctx.sparse_posterior(kind, Xu, X, y, Xs, theta, noiseless, 1e-6, ("mean", "var", "cov"))
    blocks = (k(Xu, Xu, kp, jitter=1e-6), k(Xu, X, kp, jitter=0), y, noise, k(Xu, Xs, kp, jitter=0))
    Kss = k(Xs, Xs, kp, 0.0 if noiseless else noise, jitter=1e-6)
    full = ctx.sparse_posterior_gram(*blocks, Kss, want=("mean", "var", "cov"))
    diag = ctx.sparse_posterior_gram(*blocks, np.diag(Kss).copy(), want=("mean", "var"), kss_diag=True)
    scale = np.abs(ref["cov"]).max()
    for out in (full, diag):
        assert out["info"] == 0
        np.testing.assert_allclose(out["mean"], ref["mean"], rtol=1e-9, atol=1e-9 * np.abs(ref["mean"]).max())
        np.testing.assert_allclose(out["var"], ref["var"], rtol=1e-9, atol=1e-9 * scale)
    np.testing.assert_allclose(full["cov"], ref["cov"], rtol=1e-9, atol=1e-9 * scale)


@pytest.mark.parametrize("tag", ["linrbf", "rbf"])
def test_model_posterior_matches_reference_vectors(ctx, tag):
    from gpax_b200.sparse_gp import viSparseGP
    from gpax_b200.utils import set_kernel_fn
    z = np.load(GOLDEN)

    def linrbf(X, Z, k_scale, k_length, c):
        r2 = (((X[:, None, :] - Z[None, :, :]) / k_length) ** 2).sum(-1)
        return k_scale * np.exp(-0.5 * r2) + c * X @ Z.T
    kern = set_kernel_fn(linrbf) if tag == "linrbf" else oracle.rbf_kernel
    X = z[tag + "_Xtr"]
    m = viSparseGP(X.shape[1], kern, ctx=ctx)
    m.X_train, m.y_train, m.Xu = X, z[tag + "_ytr"], z[tag + "_Xu"]
    params = {k[len(tag) + 3:]: z[k] for k in z.files if k.startswith(tag + "_p_")}
    Xs = z[tag + "_Xte"]
    for key, nl, kw in (("nl0", False, {}), ("nl1", True, {}), ("jit1e-5", False, {"jitter": 1e-5})):
        mean, cov = m.get_mvn_posterior(Xs, params, nl, **kw)
        np.testing.assert_allclose(mean, z[f"{tag}_{key}_mean"], rtol=1e-8, atol=1e-9)
        np.testing.assert_allclose(cov, z[f"{tag}_{key}_cov"], rtol=1e-8, atol=1e-9)
        pm, pv = m.predict(0, Xs, params, nl, **kw)
        np.testing.assert_allclose(pm, mean, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(pv, np.diag(cov), rtol=1e-10, atol=1e-12)
    m.KSS_CHUNK = 4
    bm, bv = m.predict_in_batches(0, Xs, batch_size=5, samples=params)
    pm, pv = m.predict(0, Xs, params)
    np.testing.assert_allclose(bm, pm, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(bv, pv, rtol=1e-12, atol=1e-12)


def _data(N=120, d=2, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (N, d))
    y = np.sin(2 * X[:, 0]) + 0.5 * X[:, -1] ** 2 + 0.05 * rng.standard_normal(N)
    return X, y


@pytest.mark.parametrize("guide", ["delta", "normal"])
def test_fit_with_callable_matches_builtin(ctx, guide):
    from gpax_b200.sparse_gp import viSparseGP
    X, y = _data()
    fits = []
    for kern in ("RBF", oracle.rbf_kernel):
        m = viSparseGP(2, kern, guide=guide, ctx=ctx)
        m.fit(0, X, y, num_steps=30, step_size=0.05, progress_bar=False, print_summary=False)
        fits.append(m)
    a, b = fits
    np.testing.assert_allclose(b.Xu, a.Xu, rtol=1e-5, atol=1e-7)
    for k in ("k_length", "k_scale", "noise"):
        np.testing.assert_allclose(b.kernel_params[k], a.kernel_params[k], rtol=1e-5)


def _oracle_bound(Xu, X, y, kp, noise, mean):
    k = oracle.rbf_kernel
    return so.elbo_gram_grad(k(Xu, Xu, kp, jitter=1e-6), k(Xu, X, kp), np.diag(k(X, X, kp, jitter=0)), y - mean, noise)[0]


@pytest.mark.parametrize("route", ["fused", "callable"])
def test_probabilistic_mean_function(ctx, route):
    from gpax_b200 import inference, priors
    from gpax_b200.sparse_gp import viSparseGP
    X, y = _data(80)
    y = y + 1.5 * X[:, 0] + 0.7
    mean_fn = lambda x, p: p["a"] * x[:, 0] + p["b"]   # noqa: E731
    mean_fn_prior = lambda: {"a": priors.sample("a", priors.Normal(0.0, 2.0)),   # noqa: E731
                             "b": priors.sample("b", priors.Normal(0.0, 2.0))}
    m = viSparseGP(2, "RBF" if route == "fused" else oracle.rbf_kernel, mean_fn=mean_fn, mean_fn_prior=mean_fn_prior, ctx=ctx)
    m.X_train, m.y_train = X, y
    Xu = X[:9] + 0.01
    lj = inference._sparse_program_log_joint(m, Xu, 1e-6) if route == "fused" else inference.SparseGramLogJoint(m, Xu, 1e-6)
    u = lj.init_u() + 0.05 * np.arange(lj.dim)
    val, g = lj(u, jacobian=False)
    vals = lj._site_values(u)
    kp = {"k_length": vals["k_length"], "k_scale": vals["k_scale"], "period": None}
    lp = lj._log_prior(u, lj._program_at(u)[3], False, want_grad=False)[0]
    assert abs(val - lp - _oracle_bound(Xu, X, y, kp, float(vals["noise"]), mean_fn(X, vals))) <= 1e-9 * abs(val)
    names = [s.name for s in lj.sites]
    h = 1e-5
    for name in ("a", "b"):   # the mean-function coordinates by central differences of the oracle bound
        kk = sum(s.size for s in lj.sites[:names.index(name)])
        e = np.zeros(lj.dim)
        e[kk] = h
        fd = []
        for uu in (u + e, u - e):
            vv = lj._site_values(uu)
            fd.append(_oracle_bound(Xu, X, y, kp, float(vv["noise"]), mean_fn(X, vv))
                      + lj._log_prior(uu, lj._program_at(uu)[3], False, want_grad=False)[0])
        np.testing.assert_allclose(g[kk], (fd[0] - fd[1]) / (2 * h), rtol=1e-5, atol=1e-6)
    m.fit(0, X, y, num_steps=40, step_size=0.05, progress_bar=False, print_summary=False)
    assert np.isfinite(m.svi.losses).all() and m.svi.losses[-1] < m.svi.losses[0]
    mean, var = m.predict(0, X[:10])
    assert np.isfinite(mean).all() and (var > 0).all()


def test_script_written_for_the_reference_runs_end_to_end(ctx):
    """set_kernel_fn kernel, mean_fn + mean_fn_prior, priors from gpax_b200.priors: fit -> predict -> EI"""
    import gpax_b200 as gpax
    from gpax_b200 import priors
    from gpax_b200.utils import set_kernel_fn

    def linrbf(X, Z, k_scale, k_length, c):
        r2 = (((X[:, None, :] - Z[None, :, :]) / k_length) ** 2).sum(-1)
        return k_scale * np.exp(-0.5 * r2) + c * X @ Z.T

    def kernel_prior():
        return {"k_length": priors.sample("k_length", priors.LogNormal(0.0, 1.0)),
                "k_scale": priors.sample("k_scale", priors.LogNormal(0.0, 1.0)),
                "c": priors.sample("c", priors.HalfNormal(1.0))}

    X, y = _data(150, 1, seed=3)
    m = gpax.viSparseGP(1, set_kernel_fn(linrbf), mean_fn=lambda x, p: p["a"] * x[:, 0],
                        mean_fn_prior=lambda: {"a": priors.sample("a", priors.Normal(0.0, 1.0))}, kernel_prior=kernel_prior)
    m.fit(0, X, y, num_steps=50, step_size=0.05, progress_bar=False, print_summary=False)
    Xs = np.linspace(-1, 1, 64)[:, None]
    mean, var = m.predict(0, Xs)
    assert mean.shape == (64,) and (var > 0).all()
    for acq in (gpax.acquisition.EI, gpax.acquisition.UCB):
        a = acq(0, m, Xs)
        assert np.asarray(a).shape == (64,) and np.isfinite(a).all()
