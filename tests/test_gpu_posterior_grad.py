"""GPU: the posterior's gradient w.r.t. the test inputs (b2gp_posterior_grad) and what is built on it: optimize_acq,
Thompson and qKG.

Each test makes a Context of its own and reads path_counts() / cache_hits() around its calls (as test_gpu_paths.py
does), so the route each result came from is witnessed:
  - N = 300 under ozaki 0: potrf_rec + trsm_rec, the derivative rows solved with [k_pX; y^T];
  - N = 2500 under ozaki 7: potrf_tall, the derivative rows ride in the factorisation;
  - a second identical single-theta call under ozaki 7: a factor-cache hit solved by trsm_tall;
  - the same under ozaki 0: a cache hit solved by trsm_rec.
dmean / dvar are held to the oracle (oracle/grad_oracle.py, pinned on CPU by central differences) at 1e-9, scaled by
cond(K) / 1e5 above cond(K) = 1e5."""
import functools

import numpy as np
import pytest
import scipy.sparse.linalg as spla

import oracle
from conftest import assert_close
from oracle import grad_oracle as gro

pytestmark = pytest.mark.gpu

RTOL = 1e-9


@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def counted(ctx, fn):
    before, hits = ctx.path_counts(), ctx.cache_hits()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}, ctx.cache_hits() - hits


def params_of(s, d):
    """hyper-parameters of draw s"""
    return {"k_length": np.linspace(0.3, 0.5, d) * (1 + 0.1 * s), "k_scale": 1.2 - 0.1 * s, "noise": 0.04 + 0.01 * s,
            "period": 1.3 + 0.2 * s}


def theta_rows(S, d):
    return np.stack([np.concatenate([p["k_length"], [p["k_scale"], p["noise"], p["period"]]])
                     for p in (params_of(s, d) for s in range(S))])


@functools.lru_cache(maxsize=4)
def problem(kernel, N, P, d, S, noiseless):
    rng = np.random.default_rng(N + 7 * P + d)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, -1]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    refs, tols = [], []
    for s in range(S):
        p = params_of(s, d)
        refs.append(gro.posterior_grad(X, y, Xn, p, kernel, noiseless))
        K = oracle.get_kernel(kernel)(X, X, p, p["noise"])
        cond = float(spla.eigsh(K, k=1, which="LA", return_eigenvectors=False, tol=1e-4)[0]) / (p["noise"] + 1e-6)
        tols.append((RTOL * max(1.0, cond / 1e5), cond))
    return X, y, Xn, refs, tols


def check(out, refs, tols, what):
    for s, (ref, (tol, cond)) in enumerate(zip(refs, tols)):
        assert out["info"][s] == 0, what
        for name, r in zip(("mean", "var", "dmean", "dvar"), ref):
            assert_close(out[name][s], r, tol, f"{name} draw {s} {what}, cond(K) = {cond:.3g}")


def same_as_posterior(ctx, kernel, X, y, Xn, theta, noiseless, out, what, fresh=False):
    """mean and var of the gradient call are those of b2gp_posterior on the same route: each row's solve does not depend
    on the others.  fresh: the plain call factors anew, as the gradient call did (otherwise it reuses the factor the
    gradient call left in the cache, as a gradient call on a cache hit does)."""
    if fresh:
        ctx.set_option("drop_factor_cache", 1)
    plain = ctx.posterior(kernel, X, y, Xn, theta, noiseless, 1e-6, ("mean", "var"))
    assert np.array_equal(out["mean"], plain["mean"]), "mean " + what
    assert np.array_equal(out["var"], plain["var"]), "var " + what
    return plain


@pytest.mark.parametrize("S", [1, 4])
@pytest.mark.parametrize("noiseless", [False, True])
@pytest.mark.parametrize("kernel", ["RBF", "Matern", "Periodic"])
def test_gradient_vs_oracle_recursive_route(ctx, kernel, noiseless, S):
    X, y, Xn, refs, tols = problem(kernel, 300, 24, 3, S, noiseless)
    theta = theta_rows(S, 3)
    ctx.set_option("ozaki", 0)
    out, moved, _ = counted(ctx, lambda: ctx.posterior_grad(kernel, X, y, Xn, theta, noiseless))
    assert moved["potrf_tall"] == 0 and moved["trsm_tall"] == 0 and moved["potrf_diag"] > 0
    check(out, refs, tols, f"{kernel} S={S} ozaki 0")
    same_as_posterior(ctx, kernel, X, y, Xn, theta, noiseless, out, f"{kernel} S={S}")


@pytest.mark.parametrize("noiseless", [False, True])
@pytest.mark.parametrize("kernel", ["RBF", "Matern", "Periodic"])
def test_gradient_tall_factorisation_then_cache_hits(ctx, kernel, noiseless):
    X, y, Xn, refs, tols = problem(kernel, 2500, 40, 2, 1, noiseless)
    theta = theta_rows(1, 2)
    run = lambda: ctx.posterior_grad(kernel, X, y, Xn, theta, noiseless)   # noqa: E731
    with ctx.options(ozaki=7):
        out, moved, hits = counted(ctx, run)
        assert moved["potrf_tall"] == 1 and hits == 0, moved
        check(out, refs, tols, f"{kernel} potrf_tall")
        same_as_posterior(ctx, kernel, X, y, Xn, theta, noiseless, out, f"{kernel} potrf_tall", fresh=True)
        out2, moved, hits = counted(ctx, run)
        assert hits == 1 and moved["trsm_tall"] == 1 and moved["potrf_tall"] == 0, moved
        check(out2, refs, tols, f"{kernel} cache hit, trsm_tall")
        same_as_posterior(ctx, kernel, X, y, Xn, theta, noiseless, out2, f"{kernel} cache hit, trsm_tall")
    with ctx.options(ozaki=0):
        out3, moved, hits = counted(ctx, run)
        assert hits == 1 and moved["trsm_tall"] == 0 and moved["potrf_tall"] == 0 and moved["potrf_diag"] == 0, moved
        check(out3, refs, tols, f"{kernel} cache hit, trsm_rec")
        same_as_posterior(ctx, kernel, X, y, Xn, theta, noiseless, out3, f"{kernel} N=2500 ozaki 0")


def test_gradient_rows_that_move_trsm_rec_onto_the_panel_route(ctx):
    """Under ozaki != 0, trsm_rec solves 1024 or more rows against a factor of at most `panel` columns by one int8 panel
    GEMM.  P + 1 = 301 rows stay on the fp64 strips, the gradient call's P + 1 + P*d = 1201 rows take the panel route:
    dmean / dvar still meet the bar, and mean / var differ from b2gp_posterior's only within the digit-plane bound."""
    X, y, Xn, refs, tols = problem("Matern", 1000, 300, 3, 2, False)
    theta = theta_rows(2, 3)
    with ctx.options(ozaki=7):
        out, moved, _ = counted(ctx, lambda: ctx.posterior_grad("Matern", X, y, Xn, theta))
        plain, moved_plain, _ = counted(ctx, lambda: ctx.posterior("Matern", X, y, Xn, theta, False, 1e-6, ("mean", "var")))
    assert moved["panel_solve"] == 2 and moved_plain["panel_solve"] == 0, (moved, moved_plain)
    check(out, refs, tols, "Matern N=1000 panel route")
    for name in ("mean", "var"):
        assert_close(out[name], plain[name], 1e-12, f"{name} panel route vs fp64 strips")


def test_gradient_with_device_pointers(ctx):
    """B2GP_FLAG_DEVICE_PTRS: inputs read from and results written to device arrays, same values as the host-pointer call"""
    import ctypes as C

    from gpax_b200 import _ffi
    X, y, Xn, refs, tols = problem("RBF", 300, 24, 3, 2, False)
    theta = theta_rows(2, 3)
    host = ctx.posterior_grad("RBF", X, y, Xn, theta)
    dX, dy, dXn, dth = (ctx.to_device(np.ascontiguousarray(a, dtype=np.float64)) for a in (X, y, Xn, theta))
    outs = {"mean": ctx.alloc((2, 24)), "var": ctx.alloc((2, 24)), "dmean": ctx.alloc((2, 24, 3)), "dvar": ctx.alloc((2, 24, 3))}
    info = np.zeros(2, dtype=np.int32)
    flags = _ffi.FLAG_DEVICE_PTRS | _ffi.OUT_MEAN | _ffi.OUT_VAR | _ffi.OUT_DMEAN | _ffi.OUT_DVAR
    ctx._check(ctx.lib.b2gp_posterior_grad(ctx.h, _ffi.KERNEL_RBF, dX.ptr, 300, dy.ptr, 0, dXn.ptr, 24, 3, 2, dth.ptr, 0, 1e-6, flags,
                                           outs["mean"].ptr, outs["var"].ptr, outs["dmean"].ptr, outs["dvar"].ptr,
                                           info.ctypes.data_as(C.c_void_p), None))
    got = {k: v.download() for k, v in outs.items()}
    got["info"] = info
    check(got, refs, tols, "device pointers")
    for name in ("mean", "var", "dmean", "dvar"):
        assert np.array_equal(got[name], host[name]), name
    for a in (dX, dy, dXn, dth, *outs.values()):
        a.free()


def test_gradient_tall_factorisation_batched_draws(ctx):
    X, y, Xn, refs, tols = problem("Matern", 2500, 40, 2, 4, False)
    theta = theta_rows(4, 2)
    with ctx.options(ozaki=7):
        out, moved, hits = counted(ctx, lambda: ctx.posterior_grad("Matern", X, y, Xn, theta))
    assert moved["potrf_tall"] == 4 and hits == 0
    check(out, refs, tols, "Matern S=4 potrf_tall")


def test_gradient_call_grows_the_buffer_around_a_cached_factor(ctx):
    """a P = 1000 posterior makes the factor; a gradient call with P = 600, d = 3 (2401 right-hand-side rows) must grow
    slot 0's buffer around it and still hit the cache"""
    X, y, Xn, refs, tols = problem("RBF", 2500, 600, 3, 1, False)
    theta = theta_rows(1, 3)
    rng = np.random.default_rng(3)
    ctx.posterior("RBF", X, y, rng.uniform(0, 1, (1000, 3)), theta, False, 1e-6, ("mean", "var"))
    out, moved, hits = counted(ctx, lambda: ctx.posterior_grad("RBF", X, y, Xn, theta))
    assert hits == 1 and moved["potrf_diag"] == 0
    check(out, refs, tols, "grown around the cached factor")


def test_failed_factorisation_gives_nan_gradients(ctx):
    X, y, Xn, _, _ = problem("RBF", 300, 24, 3, 1, False)
    theta = theta_rows(2, 3)
    theta[1, 3 + 1] = -2.0                         # negative noise: k_XX is not positive definite
    out = ctx.posterior_grad("RBF", X, y, Xn, theta)
    assert out["info"][0] == 0 and out["info"][1] > 0
    assert np.isfinite(out["dmean"][0]).all() and np.isfinite(out["dvar"][0]).all()
    for name in ("mean", "var", "dmean", "dvar"):
        assert np.isnan(out[name][1]).all(), name


def test_unsupported_flags_are_refused(ctx):
    import ctypes as C

    from gpax_b200 import _ffi
    X, y, Xn, _, _ = problem("RBF", 300, 24, 3, 1, False)
    theta = theta_rows(1, 3)
    info = np.zeros(1, dtype=np.int32)
    out = np.empty((1, 24 * 3))
    for bad in (_ffi.FLAG_F32, _ffi.OUT_COV, _ffi.OUT_SAMPLE):
        rc = ctx.lib.b2gp_posterior_grad(ctx.h, 0, _ffi._ptr(X), 300, _ffi._ptr(y), 0, _ffi._ptr(Xn), 24, 3, 1, _ffi._ptr(theta), 0,
                                         1e-6, _ffi.OUT_DMEAN | bad, None, None, _ffi._ptr(out), None, info.ctypes.data_as(C.c_void_p),
                                         None)
        assert rc == -4, bad


# ------------------------------------------------------------------ optimize_acq, Thompson, qKG
class FakeMCMC:
    def __init__(self, samples):
        self.samples = samples

    def get_samples(self, group_by_chain=False):
        return self.samples


def mcmc_samples(d, S=3):
    return {"k_length": np.stack([params_of(s, d)["k_length"] * 3 for s in range(S)]),
            "k_scale": np.array([params_of(s, d)["k_scale"] for s in range(S)]) * 10,
            "noise": np.array([params_of(s, d)["noise"] for s in range(S)]) * 0.1}


def bo_models(ctx, d):
    from gpax_b200 import ExactGP, viGP
    rng = np.random.default_rng(11 + d)
    if d == 1:
        X = rng.uniform(-2, 2, size=(4,))              # the reference's tests/test_optimize_acq.py problem
        y = X ** 3
    else:
        X = rng.uniform(-2, 2, size=(12, d))
        y = (X ** 3).sum(1) - X.prod(1)
    m = ExactGP(d, "RBF", ctx=ctx)
    m.X_train, m.y_train, m.mcmc = X, y, FakeMCMC(mcmc_samples(d))
    v = viGP(d, "RBF", ctx=ctx)
    v.X_train, v.y_train = X, y
    v.kernel_params = {k: np.asarray(a)[0] for k, a in mcmc_samples(d).items()}
    return {"mcmc": m, "vi": v}


def count_calls(ctx):
    """wrap the context's posterior entry points to count the calls made through them"""
    calls = {"n": 0}
    for name in ("posterior", "posterior_grad"):
        fn = getattr(ctx, name)

        def wrapped(*a, _fn=fn, **k):
            calls["n"] += 1
            return _fn(*a, **k)
        setattr(ctx, name, wrapped)
    return calls


@pytest.mark.parametrize("model_kind", ["mcmc", "vi"])
@pytest.mark.parametrize("acq_name", ["EI", "UCB"])
@pytest.mark.parametrize("d", [1, 2])
def test_optimize_acq_end_to_end(ctx, d, acq_name, model_kind):
    from gpax_b200 import acquisition as acq, prng
    model = bo_models(ctx, d)[model_kind]
    acq_fn = getattr(acq, acq_name)
    key = prng.PRNGKey(5)
    lb, ub = (-2.0, 2.0) if d == 1 else ([-2.0] * d, [2.0] * d)
    kw = {"noiseless": True}

    ctx.set_option("drop_factor_cache", 1)
    calls = count_calls(ctx)
    hits0 = ctx.cache_hits()
    x = acq.optimize_acq(key, model, acq_fn, 5, lb, ub, **kw)
    n_calls, hits = calls["n"], ctx.cache_hits() - hits0
    assert x.shape == (() if d == 1 else (d,))
    assert np.all(x >= np.asarray(lb)) and np.all(x <= np.asarray(ub))
    lbA, ubA = acq.ensure_array(lb), acq.ensure_array(ub)
    guesses = prng.uniform(key, (5, d), np.float32, lbA.astype(np.float32), ubA.astype(np.float32))
    best0 = np.max(acq_fn(key, model, guesses, **kw))
    xq = np.asarray(x, np.float64).reshape(1, d)
    assert acq_fn(key, model, xq, **kw)[0] >= best0 - 1e-12 * abs(best0)
    if model_kind == "vi":
        assert hits == n_calls - 1, (hits, n_calls)        # one factorisation for the whole optimisation

    # the analytic gradient against central differences of the GPU-evaluated acquisition, at an interior point
    f = acq._analytic_objective(acq_name, key, model, d, kw)
    x0 = np.linspace(-0.7, 0.4, d)
    val, grad = f(x0)
    assert np.isclose(val, acq_fn(key, model, x0[None], **kw)[0], rtol=1e-12, atol=0), "value of the gradient path"
    h, fd = 1e-5, np.empty(d)
    for k in range(d):
        e = np.zeros(d)
        e[k] = h
        fd[k] = (acq_fn(key, model, (x0 + e)[None], **kw)[0] - acq_fn(key, model, (x0 - e)[None], **kw)[0]) / (2 * h)
    np.testing.assert_allclose(grad, fd, rtol=1e-5, atol=1e-5 * np.abs(fd).max())


def test_optimize_acq_without_an_analytic_gradient_takes_finite_differences(ctx):
    """a penalty (or any acquisition without a closed-form gradient) goes to L-BFGS-B without one"""
    from gpax_b200 import acquisition as acq
    model = bo_models(ctx, 2)["vi"]
    assert acq._analytic_kind(acq.EI, model, {"penalty": "inverse_distance"}) is None
    assert acq._analytic_kind(acq.KG, model, {}) is None
    assert acq._analytic_kind(acq.EI, model, {}) == "EI"
    x = acq.optimize_acq(0, model, acq.EI, 4, [-2.0, -2.0], [2.0, 2.0], penalty="inverse_distance",
                         recent_points=np.zeros((1, 2)))
    assert x.shape == (2,) and np.all(np.abs(x) <= 2.0)


def test_thompson_is_predict_on_the_draw_randint_picks(ctx):
    from gpax_b200 import acquisition as acq, prng
    model = bo_models(ctx, 1)["mcmc"]
    Xn = np.random.default_rng(0).standard_normal(12)
    key = prng.PRNGKey(9)
    t = acq.Thompson(key, model, Xn)
    assert t.squeeze().shape == (12,)                    # the reference's tests/test_acq.py:93-103
    idx = prng.randint(key, (1,), 0, 3)
    one = {k: np.asarray(v)[idx] for k, v in model.get_samples().items()}
    np.testing.assert_array_equal(t, model.predict(key, Xn, one, 1)[1])
    t4 = acq.Thompson(key, model, Xn, n=4)
    np.testing.assert_allclose(t4, model.predict(key, Xn, one, 4)[1].mean(1).squeeze(), rtol=0, atol=0)
    with pytest.raises(AttributeError):
        acq.Thompson(key, bo_models(ctx, 1)["vi"], Xn)


@pytest.mark.parametrize("maximize_distance", [False, True])
def test_qkg_rows_are_kg_of_the_subsampled_draws(ctx, maximize_distance):
    from gpax_b200 import acquisition as acq, prng
    model = bo_models(ctx, 1)["mcmc"]
    Xn = np.linspace(-2, 2, 10)
    key = prng.PRNGKey(4)
    q = acq.qKG(key, model, Xn, n=3, subsample_size=2, maximize_distance=maximize_distance, n_evals=3)
    assert q.shape == (2, 10) and np.isfinite(q).all()
    if not maximize_distance:
        sub = acq._subsample(model.get_samples(), 2, key)
        rows = [acq.kg(model, Xn, {k: np.asarray(v)[s] for k, v in sub.items()}, key, 3, False, False) for s in range(2)]
        np.testing.assert_array_equal(q, np.stack(rows))
    with pytest.raises(ValueError):
        acq.qKG(key, bo_models(ctx, 1)["vi"], Xn)
