"""iBNN / vi_iBNN on the GPU: b2gp_posterior(_batch) and b2gp_mll(_v) on the NNGP kinds against the NumPy oracle
(oracle/ibnn_oracle.py), the variance epilogue against diag(cov), the factor cache, the routes (fp64 tall panels, int8 digit
planes, the new gradient kernel's path counter), determinism, the refusals, and the two models end to end."""
import numpy as np
import pytest

from oracle import gp_oracle as go
from oracle import ibnn_oracle as io

pytestmark = pytest.mark.gpu

KIND = {"erf": 3, "relu": 4}
JIT = 1e-6
PARAMS = {"var_b": 0.6, "var_w": 1.7, "noise": 0.05}


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def _theta(d, depth, p=PARAMS):
    return np.r_[np.full(d, float(depth)), p["var_w"], p["noise"], p["var_b"]]


def _problem(N, P, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1.5, 1.5, (N, d))
    y = np.sin(2 * X[:, 0]) + 0.3 * X[:, -1] ** 2 + 0.05 * rng.standard_normal(N)
    return X, y, rng.uniform(-1.5, 1.5, (P, d))


def _close(got, ref, tol, what, scale=None):
    """max |got - ref| <= tol * scale; scale defaults to max |ref|.  A posterior covariance is k_pp - V^T V, so its
    rounding error is relative to the prior covariance k_pp, which is the scale the callers pass for cov and var."""
    scale = max(np.abs(ref).max(), 1e-300) if scale is None else scale
    err = np.abs(np.asarray(got, dtype=np.float64) - ref).max()
    assert err <= tol * scale, f"{what}: max error {err:.3e} vs scale {scale:.3e}"


def _prior_scale(Xn, act, depth, p=PARAMS):
    """max |k_pp|: the scale of the terms the posterior covariance is the difference of"""
    return np.abs(io.kernel(Xn, Xn, p, p["noise"], JIT, act, depth)).max()


def _cond(X, act, depth, p=PARAMS):
    return np.linalg.cond(io.kernel(X, X, p, p["noise"], JIT, act, depth))


def _counts(ctx, fn):
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


# ------------------------------------------------------------------ posterior
@pytest.mark.parametrize("noiseless", [False, True])
@pytest.mark.parametrize("d", [1, 5, 64])
@pytest.mark.parametrize("depth", [0, 1, 3])
@pytest.mark.parametrize("act", ["erf", "relu"])
def test_posterior_matches_oracle(ctx, act, depth, d, noiseless):
    X, y, Xn = _problem(200, 37, d, seed=depth * 10 + d)
    out = ctx.posterior(KIND[act], X, y, Xn, _theta(d, depth)[None], noiseless, JIT, want=("mean", "var", "cov"))
    assert out["info"][0] == 0
    rmean, rcov = io.posterior(X, y, Xn, PARAMS, act, depth, noiseless)
    c = f"cond(K) = {_cond(X, act, depth):.2e}"
    ps = _prior_scale(Xn, act, depth)
    _close(out["mean"][0], rmean, 1e-9, "mean, " + c)
    _close(out["cov"][0], rcov, 1e-9, "cov, " + c, max(np.abs(rcov).max(), ps))
    _close(out["var"][0], np.diag(rcov), 1e-9, "var, " + c, max(np.abs(rcov).max(), ps))
    v, dc = out["var"][0], np.diag(out["cov"][0])
    _close(v, dc, 1e-12, "var vs diag(cov)", max(np.abs(dc).max(), ps))


@pytest.mark.parametrize("act", ["erf", "relu"])
def test_posterior_samples_with_injected_eps(ctx, act):
    d, depth, S, n = 3, 2, 3, 4
    X, y, Xn = _problem(150, 20, d, seed=5)
    p = [dict(PARAMS, var_w=PARAMS["var_w"] * (1 + 0.2 * s)) for s in range(S)]
    theta = np.stack([_theta(d, depth, ps) for ps in p])
    eps = np.random.default_rng(1).standard_normal((S, n, 20))
    out = ctx.posterior(KIND[act], X, y, Xn, theta, False, JIT, want=("mean",), eps=eps)
    for s in range(S):
        rmean, rcov = io.posterior(X, y, Xn, p[s], act, depth)
        _close(out["mean"][s], rmean, 1e-9, f"mean draw {s}")
        ref = rmean[None] + eps[s] @ np.linalg.cholesky(rcov).T
        _close(out["y_sampled"][s], ref, 1e-8, f"samples draw {s}")


def test_posterior_batch_per_member_inputs(ctx):
    d, depth, S = 4, 3, 3
    probs = [_problem(120, 16, d, seed=20 + s) for s in range(S)]
    Xtr = np.stack([pr[0] for pr in probs])
    ys = np.stack([pr[1] for pr in probs])
    Xn = np.stack([pr[2] for pr in probs])
    theta = np.stack([_theta(d, depth)] * S)
    out = ctx.posterior(KIND["relu"], Xtr, ys, Xn, theta, False, JIT, want=("mean", "var"))
    for s in range(S):
        rmean, rcov = io.posterior(Xtr[s], ys[s], Xn[s], PARAMS, "relu", depth)
        _close(out["mean"][s], rmean, 1e-9, f"mean member {s}")
        _close(out["var"][s], np.diag(rcov), 1e-9, f"var member {s}")


def test_posterior_tall_fp64_route(ctx):
    N, P, d, depth = 8192, 64, 3, 1
    X, y, Xn = _problem(N, P, d, seed=7)
    out, c = _counts(ctx, lambda: ctx.posterior(KIND["erf"], X, y, Xn, _theta(d, depth)[None], False, JIT, want=("mean", "cov")))
    assert c["potrf_tall_fp64"] == 1, c
    kern = lambda A, B, p, noise=0, jitter=1e-6: io.kernel(A, B, p, noise, jitter, "erf", depth)   # noqa: E731
    rmean, rcov = go.exact_posterior_chol(X, y, Xn, PARAMS, kern)
    _close(out["mean"][0], rmean, 1e-9, "mean (N = 8192)")
    _close(out["cov"][0], rcov, 1e-9, "cov (N = 8192)")


def test_posterior_auto_digit_planes(ctx):
    N, P, d, depth = 2300, 40, 5, 2
    X, y, Xn = _problem(N, P, d, seed=8)
    with ctx.options(ozaki=-1):
        out, c = _counts(ctx, lambda: ctx.posterior(KIND["relu"], X, y, Xn, _theta(d, depth)[None], False, JIT, want=("mean", "var")))
    assert c["oz_mma"] > 0, c
    rmean, rcov = io.posterior(X, y, Xn, PARAMS, "relu", depth)
    cd = f"cond(K) = {_cond(X, 'relu', depth):.2e}"
    _close(out["mean"][0], rmean, 1e-9, "mean, ozaki = -1, " + cd)
    _close(out["var"][0], np.diag(rcov), 1e-9, "var, ozaki = -1, " + cd)


def test_factor_cache_keys_on_depth_and_activation(ctx):
    d = 2
    X, y, Xn = _problem(300, 10, d, seed=9)
    ctx.set_option("drop_factor_cache", 1)
    call = lambda act, depth: ctx.posterior(KIND[act], X, y, Xn, _theta(d, depth)[None], False, JIT, want=("mean", "var"))  # noqa: E731
    h0 = ctx.cache_hits()
    a = call("erf", 2)
    b = call("erf", 2)
    assert ctx.cache_hits() == h0 + 1
    np.testing.assert_array_equal(a["mean"], b["mean"])
    for act, depth in (("erf", 3), ("relu", 3), ("relu", 2)):
        out = call(act, depth)
        assert ctx.cache_hits() == h0 + 1, (act, depth)
        rmean, rcov = io.posterior(X, y, Xn, PARAMS, act, depth)
        _close(out["mean"][0], rmean, 1e-9, f"mean after a miss ({act}, depth {depth})")
        _close(out["var"][0], np.diag(rcov), 1e-9, f"var after a miss ({act}, depth {depth})")


# ------------------------------------------------------------------ likelihood
@pytest.mark.parametrize("N", [300, 2300])
@pytest.mark.parametrize("d", [1, 5, 64])
@pytest.mark.parametrize("act", ["erf", "relu"])
def test_mll_matches_oracle(ctx, act, d, N):
    depth = 3
    X, y, _ = _problem(N, 1, d, seed=N + d)
    th = _theta(d, depth)
    (val, g, _, info), c = _counts(ctx, lambda: ctx.mll(KIND[act], X, y, th, JIT))
    assert info == 0 and c["mll_nngp_grad"] == 1, c
    rv, rg = io.mll_grad(X, y, PARAMS, act, depth)
    cd = f"cond(K) = {_cond(X, act, depth):.2e}"
    assert abs(val - rv) <= 1e-9 * abs(rv), f"value {val} vs {rv}, {cd}"
    assert np.all(g[:d] == 0.0)
    _close(g[d:], rg, 1e-8, "grad, " + cd)


@pytest.mark.parametrize("depth", [0, 1])
def test_mll_shallow_depths(ctx, depth):
    d = 3
    X, y, _ = _problem(400, 1, d, seed=11)
    val, g, _, info = ctx.mll(KIND["relu"], X, y, _theta(d, depth), JIT)
    rv, rg = io.mll_grad(X, y, PARAMS, "relu", depth)
    assert info == 0 and abs(val - rv) <= 1e-9 * abs(rv)
    _close(g[d:], rg, 1e-8, f"grad, depth {depth}")


def test_mll_v_with_noise_vector(ctx):
    d, depth = 4, 2
    X, y, _ = _problem(500, 1, d, seed=12)
    nv = np.random.default_rng(3).uniform(0.01, 0.1, 500)
    val, g, _, info, gnv = ctx.mll(KIND["erf"], X, y, _theta(d, depth), JIT, noise_vec=nv)
    rv, rg = io.mll_grad(X, y, PARAMS, "erf", depth, noise_vec=nv)
    assert info == 0 and abs(val - rv) <= 1e-9 * abs(rv)
    _close(g[d:], rg, 1e-8, "grad with noise_vec")
    assert gnv.shape == (500,) and np.all(np.isfinite(gnv))


def test_mll_is_deterministic(ctx):
    d = 5
    X, y, _ = _problem(1500, 1, d, seed=13)
    a = ctx.mll(KIND["relu"], X, y, _theta(d, 3), JIT)
    b = ctx.mll(KIND["relu"], X, y, _theta(d, 3), JIT)
    assert a[0] == b[0]
    np.testing.assert_array_equal(a[1], b[1])


# ------------------------------------------------------------------ refusals
def test_refusals(ctx):
    from gpax_b200._ffi import B200GPError
    d = 2
    X, y, Xn = _problem(64, 8, d, seed=14)
    th = _theta(d, 2)
    task = np.zeros(64, dtype=np.int32)
    for kind in (3, 4):
        calls = [
            lambda: ctx.posterior_grad(kind, X, y, Xn, th[None]),
            lambda: ctx.posterior_multitask(kind, X, task, y, Xn, task[:8], np.ones((1, 1, d + 2)), np.ones((1, 1, 1, 1)),
                                            np.full((1, 1), 0.1)),
            lambda: ctx.mll_multitask(kind, X, task, y, np.ones((1, d + 2)), np.ones((1, 1, 1)), np.full(1, 0.1)),
            lambda: ctx.sparse_posterior(kind, X[:8], X, y, Xn, th),
            lambda: ctx.sparse_elbo(kind, X[:8], X, y, th),
            lambda: ctx.dkl_mll(kind, X, y, [], 0, np.zeros(0), th),
            lambda: ctx.mtdkl_mll(kind, X, task, y, [], 0, np.zeros(0), np.ones((1, d + 2)), np.ones((1, 1, 1)), np.full(1, 0.1)),
        ]
        for i, f in enumerate(calls):
            with pytest.raises(B200GPError, match="error -1:"):
                f()
    for bad, code in ((17.0, -4), (2.5, -1), (-1.0, -1)):
        t = th.copy()
        t[:d] = bad
        with pytest.raises(B200GPError, match=f"error {code}:"):
            ctx.mll(3, X, y, t, JIT)
        with pytest.raises(B200GPError, match=f"error {code}:"):
            ctx.posterior(4, X, y, Xn, t[None], False, JIT, want=("mean",))
    ctx.mll(3, X, y, th, JIT)                        # the context is usable after the refusals


# ------------------------------------------------------------------ models
def _ref_data():
    rng = np.random.default_rng(0)
    X = np.linspace(1, 2, 8) + 0.1 * rng.standard_normal(8)     # the reference's own fixture (tests/test_ibnn.py)
    return X, 10 * X ** 2


@pytest.mark.parametrize("act", ["erf", "relu"])
def test_ibnn_fit_and_predict(act):
    from gpax_b200 import iBNN
    X, y = _ref_data()
    m = iBNN(1, depth=3, activation=act)
    m.fit(0, X, y, num_warmup=200, num_samples=200, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert set(s) == {"var_b", "var_w", "noise"} and s["var_b"].shape == (200,)
    Xn = np.linspace(0.8, 2.2, 17)
    mean, ys = m.predict(1, Xn, n=2)
    assert mean.shape == (17,) and ys.shape == (200, 2, 17) and np.all(np.isfinite(ys))
    p = {k: v[0] for k, v in s.items()}
    mu, cov = m.get_mvn_posterior(Xn, p)
    # a fitted noise can be small: the Cholesky-based oracle is the arbiter, and the tolerance follows cond(K)
    kern = lambda A, B, q, noise=0, jitter=1e-6: io.kernel(A, B, q, noise, jitter, act, 3)   # noqa: E731
    rmu, rcov = go.exact_posterior_chol(X[:, None], y, Xn[:, None], p, kern)
    cond = _cond(X[:, None], act, 3, p)
    tol = max(1e-9, 100 * cond * np.finfo(float).eps)
    _close(mu, rmu, tol, f"get_mvn_posterior mean, cond(K) = {cond:.2e}")
    _close(cov, rcov, tol, f"get_mvn_posterior cov, cond(K) = {cond:.2e}", max(np.abs(rcov).max(), _prior_scale(Xn[:, None], act, 3, p)))
    ym, yb = m.predict_in_batches(1, Xn, batch_size=5, samples={k: v[:4] for k, v in s.items()}, n=1)
    assert ym.shape == (17,) and yb.shape == (4, 1, 17)
    prior = m.sample_from_prior(2, Xn, num_samples=3)
    assert prior.shape == (3, 17) and np.all(np.isfinite(prior))


@pytest.mark.parametrize("act", ["erf", "relu"])
def test_vi_ibnn_fit_and_predict(act):
    from gpax_b200 import vi_iBNN
    X, y = _ref_data()
    m = vi_iBNN(1, depth=3, activation=act)
    m.fit(0, X, y, num_steps=300, step_size=5e-3, progress_bar=False, print_summary=False)
    p = m.get_samples()
    assert set(p) == {"var_b", "var_w", "noise"}
    Xn = np.linspace(0.8, 2.2, 17)
    mean, var = m.predict(0, Xn)
    assert mean.shape == var.shape == (17,) and np.all(np.isfinite(mean)) and np.all(var > 0)
    rmu, rvar = io.vi_predict(X[:, None], y, Xn[:, None], p, act, 3)
    _close(mean, rmu, 1e-9, "vi predict mean")
    _close(var, rvar, 1e-9, "vi predict var")


@pytest.mark.parametrize("cls_name", ["iBNN", "vi_iBNN"])
def test_svi_objective_gradient_matches_the_oracle(cls_name):
    import gpax_b200
    from gpax_b200.inference import make_log_joint
    X, y = _ref_data()
    m = getattr(gpax_b200, cls_name)(1, depth=2, activation="relu")
    m.X_train, m.y_train = X[:, None], y
    lj = make_log_joint(m)
    u = np.array([-0.2, 0.4, -1.0])
    th = lj.theta_of(u)
    p = {"var_w": th[1], "noise": th[2], "var_b": th[3]}
    for jac in (False, True):
        v, g = lj(u, jac)
        rv, rg = io.mll_grad(X[:, None], y, p, "relu", 2)
        ref = np.zeros(3)
        for k, (pr, i) in enumerate(zip(lj.priors, (3, 1, 2))):
            t = th[i]
            dt = float(pr.dtheta_du(u[k]))
            rv += float(pr.log_prob(t)) + (float(pr.log_abs_jac(u[k])) if jac else 0.0)
            ref[k] = rg[i - 1] / t * dt + float(pr.dlog_prob(t)) * dt + (float(pr.dlog_abs_jac(u[k])) if jac else 0.0)
        assert abs(v - rv) <= 1e-9 * abs(rv)
        _close(g, ref, 1e-8, f"log joint gradient (jacobian={jac})")


def test_float32_io():
    from gpax_b200 import iBNN, vi_iBNN
    X, y = _ref_data()
    Xn = np.linspace(0.8, 2.2, 9).astype(np.float32)
    p = {"var_b": 0.5, "var_w": 2.0, "noise": 0.1}
    for cls in (iBNN, vi_iBNN):
        m = cls(1, depth=2)
        m.X_train, m.y_train = X.astype(np.float32)[:, None], y.astype(np.float32)
        mu, cov = m.get_mvn_posterior(Xn, p)
        assert mu.dtype == cov.dtype == np.float32
        rmu, rcov = io.posterior(X.astype(np.float32)[:, None].astype(np.float64), y.astype(np.float32), Xn[:, None], p, "erf", 2)
        _close(mu, rmu, 1e-5, "float32 mean")
    m = vi_iBNN(1, depth=2)
    m.X_train, m.y_train = X.astype(np.float32)[:, None], y.astype(np.float32)
    mean, var = m.predict(0, Xn, samples=p)
    assert mean.dtype == var.dtype == np.float32


def test_optimize_acq_on_a_fitted_ibnn():
    from gpax_b200 import acquisition as acq
    from gpax_b200 import iBNN
    X, y = _ref_data()
    m = iBNN(1, depth=2)
    m.fit(0, X, y, num_warmup=100, num_samples=50, progress_bar=False, print_summary=False)
    x = acq.optimize_acq(0, m, acq.EI, 4, np.array([0.5]), np.array([2.5]))
    assert np.all(np.isfinite(x)) and 0.5 <= float(np.asarray(x).reshape(-1)[0]) <= 2.5
