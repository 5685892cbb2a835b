"""GPU: the posterior of viDKL / DKL and its gradient w.r.t. the raw test inputs (b2gp_dkl_posterior_grad), and
optimize_acq on those models.

- against the oracle (tests/dkl_grad_oracle.py, pinned on CPU by central differences) at 1e-9, scaled by cond(K) / 1e5
  above cond(K) = 1e5, over both activations, the three kernels, S in {1, 4}, P in {1, 17} and D in {1, 6, 300} (300
  spans several VJP_TILE tiles of the input dimension), with a hidden layer wider than a CTA and one too wide for the
  kernel's shared-memory buffers;
- against the existing calls: mean / var are b2gp_posterior's on b2gp_mlp_forward's embeddings, bit for bit on the same
  route, and n_layers = 0 is b2gp_posterior_grad;
- the factor cache: a repeated single-weight-set call solves against the cached factor, and optimize_acq on a viDKL
  factors once, for its initial guesses;
- optimize_acq end to end on a viDKL and a DKL with hand-set weights and draws;
- refusals, failed draws and determinism."""
import ctypes as C

import numpy as np
import pytest

import oracle
from conftest import assert_close
from dkl_grad_oracle import posterior_grad as oracle_grad
from oracle import dkl_oracle as dko

pytestmark = pytest.mark.gpu

RTOL = 1e-9
ACT = {"relu": 0, "tanh": 1}


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


def network(D, widths, S, seed):
    """flat weight sets [S, P]: draw s perturbs draw 0"""
    from gpax_b200._ffi import _mlp_nparams
    rng = np.random.default_rng(seed)
    base, i = [], D
    for w in widths:
        base += [rng.standard_normal(i * w) / np.sqrt(i), 0.3 * rng.standard_normal(w)]
        i = w
    flat = np.concatenate(base)
    assert flat.size == _mlp_nparams(D, widths)
    return np.stack([flat * (1 + 0.05 * s) + 0.01 * s for s in range(S)])


def theta_rows(S, dz):
    return np.stack([np.concatenate([np.linspace(0.8, 1.2, dz) * (1 + 0.1 * s), [1.2 - 0.1 * s, 0.04 + 0.01 * s, 1.7 + 0.2 * s]])
                     for s in range(S)])


def params_of(th, dz):
    return {"k_length": th[:dz], "k_scale": th[dz], "noise": th[dz + 1], "period": th[dz + 2]}


def kink_free_points(rng, P, D, flats, widths, act, margin=1e-6):
    """test inputs whose hidden ReLU pre-activations all lie at least `margin` from the kink under every weight set:
    there the mask does not depend on the summation order"""
    rows = []
    while len(rows) < P:
        x = rng.uniform(-1, 1, (1, D))
        ok = True
        for flat in flats:
            h = x
            for W, b in dko.unflatten(flat, D, widths)[:-1]:
                pre = h @ W + b
                ok &= act == "tanh" or bool(np.abs(pre).min() > margin)
                h = dko._act(pre, act)
        if ok:
            rows.append(x[0])
    return np.array(rows)


def problem(kind, act, N, P, D, S, widths, seed=0):
    rng = np.random.default_rng(seed + D + 7 * P + 31 * S)
    X = rng.uniform(-1, 1, (N, D))
    y = np.sin(2 * X[:, 0]) * np.cos(X[:, -1]) + 0.05 * rng.standard_normal(N)
    flats = network(D, widths, S, seed + D)
    Xn = kink_free_points(rng, P, D, flats, widths, act)
    theta = theta_rows(S, widths[-1])
    return X, y, Xn, flats, theta


def oracle_check(out, kind, act, X, y, Xn, flats, theta, widths, noiseless, what):
    D, dz = X.shape[1], widths[-1]
    for s in range(theta.shape[0]):
        layers = dko.unflatten(flats[s], D, widths)
        p = params_of(theta[s], dz)
        z = dko.mlp_forward(X, layers, act)[-1]
        K = oracle.get_kernel(kind)(z, z, p, p["noise"])
        cond = float(np.linalg.eigvalsh(K)[-1]) / (p["noise"] + 1e-6)
        tol = RTOL * max(1.0, cond / 1e5)
        assert out["info"][s] == 0, what
        for name, r in zip(("mean", "var", "dmean", "dvar"), oracle_grad(kind, X, y, Xn, layers, act, p, noiseless)):
            assert_close(out[name][s], r, tol, f"{name} draw {s} {what}, cond(K) = {cond:.3g}")


@pytest.mark.parametrize("D", [1, 6, 300])
@pytest.mark.parametrize("P", [1, 17])
@pytest.mark.parametrize("S", [1, 4])
@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_matches_oracle(ctx, act, kind, S, P, D):
    widths = [300, 16, 2] if D == 6 else [32, 2]          # 300: a hidden layer wider than the 256-thread CTA
    X, y, Xn, flats, theta = problem(kind, act, 200, P, D, S, widths)
    noiseless = P == 17
    out = ctx.dkl_posterior_grad(kind, X, y, Xn, widths, ACT[act], flats, theta, noiseless)
    oracle_check(out, kind, act, X, y, Xn, flats, theta, widths, noiseless, f"{act} {kind} S={S} P={P} D={D}")


@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_hidden_layer_wider_than_shared_memory(ctx, act):
    """2 x 2 x 1600 doubles of G buffers exceed the kernel's shared-memory budget: the same code runs on global scratch"""
    widths = [1600, 40, 3]
    X, y, Xn, flats, theta = problem("Matern", act, 150, 5, 70, 2, widths, seed=3)
    out = ctx.dkl_posterior_grad("Matern", X, y, Xn, widths, ACT[act], flats, theta)
    oracle_check(out, "Matern", act, X, y, Xn, flats, theta, widths, False, f"{act} wide hidden layer")


@pytest.mark.parametrize("S", [1, 4])
@pytest.mark.parametrize("kind", ["RBF", "Periodic"])
def test_mean_var_are_the_posterior_on_the_embeddings(ctx, kind, S):
    widths = [24, 12, 2]
    X, y, Xn, flats, theta = problem(kind, "relu", 300, 17, 6, S, widths, seed=5)
    ctx.set_option("drop_factor_cache", 1)
    out = ctx.dkl_posterior_grad(kind, X, y, Xn, widths, 0, flats, theta)
    Ztr = ctx.mlp_forward(X, widths, 0, flats)
    Zn = ctx.mlp_forward(Xn, widths, 0, flats)
    plain = ctx.posterior(kind, Ztr[0] if S == 1 else Ztr, y, Zn[0] if S == 1 else Zn, theta, False, 1e-6, ("mean", "var"))
    for name in ("mean", "var"):
        assert np.array_equal(out[name], plain[name]), name
    # a cache hit on the plain call's factor, and the plain call on the same hit: the same bits again
    if S == 1:
        out2, _, hits = counted(ctx, lambda: ctx.dkl_posterior_grad(kind, X, y, Xn, widths, 0, flats, theta))
        plain2, _, hits2 = counted(ctx, lambda: ctx.posterior(kind, Ztr[0], y, Zn[0], theta, False, 1e-6, ("mean", "var")))
        assert hits == 1 and hits2 == 1
        for name in ("mean", "var"):
            assert np.array_equal(out2[name], plain2[name]), name
        for name in ("dmean", "dvar"):
            assert_close(out2[name], out[name], 1e-12, name)


@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
def test_no_layers_is_posterior_grad(ctx, kind):
    rng = np.random.default_rng(2)
    X, Xn = rng.uniform(-1, 1, (250, 3)), rng.uniform(-1, 1, (9, 3))
    y = np.sin(3 * X[:, 0]) + 0.1 * rng.standard_normal(250)
    theta = theta_rows(2, 3)
    ctx.set_option("drop_factor_cache", 1)
    got = ctx.dkl_posterior_grad(kind, X, y, Xn, [], 0, np.zeros(0), theta)
    ctx.set_option("drop_factor_cache", 1)
    ref = ctx.posterior_grad(kind, X, y, Xn, theta)
    for name in ("mean", "var", "dmean", "dvar"):
        assert np.array_equal(got[name], ref[name]), name


@pytest.mark.parametrize("N,ozaki", [(300, 0), (2500, 7)])
def test_single_weight_set_reuses_the_cached_factor(ctx, N, ozaki):
    widths = [32, 32, 2]
    X, y, Xn, flats, theta = problem("RBF", "relu", N, 3, 8, 1, widths, seed=9)
    potrf = ("potrf_diag", "potrf_tall", "potrf_tall_fp64")
    run = lambda: ctx.dkl_posterior_grad("RBF", X, y, Xn, widths, 0, flats, theta)   # noqa: E731
    with ctx.options(ozaki=ozaki):
        ctx.set_option("drop_factor_cache", 1)
        out, moved, hits = counted(ctx, run)
        assert hits == 0 and sum(moved[k] for k in potrf) > 0, moved
        out2, moved, hits = counted(ctx, run)
        assert hits == 1 and all(moved[k] == 0 for k in potrf), moved
        if ozaki:
            assert moved["trsm_tall"] == 1, moved
    # ozaki 7: the hit solves by trsm_tall's digit planes, the first call inside the factorisation -- equal within the
    # parity bar; ozaki 0: the same fp64 solves on both
    for name in ("dmean", "dvar"):
        assert_close(out2[name], out[name], 1e-9 if ozaki else 1e-12, name)


# ------------------------------------------------------------------ optimize_acq on viDKL / DKL
class FakeMCMC:
    def __init__(self, samples):
        self.samples = samples

    def get_samples(self, group_by_chain=False):
        return self.samples


def bo_models(ctx, D=3):
    """a viDKL (ReLU 64-64-2) and a DKL (tanh 8-6-2, three draws) with hand-set weights on a cubic test function"""
    from gpax_b200 import DKL, viDKL
    rng = np.random.default_rng(21)
    X = rng.uniform(-2, 2, size=(30, D))
    y = (X ** 3).sum(1) / 8 - X.prod(1) / 4
    v = viDKL(D, 2, "RBF", ctx=ctx)
    v.X_train, v.y_train = X, y
    v.nn_params = v.from_flat(network(D, v.widths, 1, 4)[0] * 0.7)
    v.kernel_params = {"k_length": np.array([0.9, 1.1]), "k_scale": np.array(1.5), "noise": np.array(0.02)}
    m = DKL(D, 2, "Matern", hidden_dim=[8, 6], ctx=ctx)
    m.X_train, m.y_train = X, y
    S = 3
    samples = m.from_flat(network(D, m.widths, S, 6))
    samples.update({"k_length": np.stack([np.array([0.8, 1.2]) * (1 + 0.1 * s) for s in range(S)]),
                    "k_scale": np.array([1.4, 1.2, 1.0]), "noise": np.array([0.02, 0.03, 0.05])})
    m.mcmc = FakeMCMC(samples)
    return {"vidkl": v, "dkl": m}


def count_grad_calls(ctx):
    calls = {"n": 0}
    fn = ctx.dkl_posterior_grad

    def wrapped(*a, **k):
        calls["n"] += 1
        return fn(*a, **k)
    ctx.dkl_posterior_grad = wrapped
    return calls


@pytest.mark.parametrize("model_kind", ["vidkl", "dkl"])
@pytest.mark.parametrize("acq_name", ["EI", "UCB"])
def test_optimize_acq_end_to_end(ctx, acq_name, model_kind):
    from gpax_b200 import acquisition as acq, prng
    D = 3
    model = bo_models(ctx, D)[model_kind]
    acq_fn = getattr(acq, acq_name)
    key = prng.PRNGKey(5)
    lb, ub = [-2.0] * D, [2.0] * D
    kw = {"noiseless": True}
    assert acq._analytic_kind(acq_fn, model, kw) == acq_name

    ctx.set_option("drop_factor_cache", 1)
    calls = count_grad_calls(ctx)
    hits0 = ctx.cache_hits()
    x = acq.optimize_acq(key, model, acq_fn, 8, lb, ub, **kw)
    n_grad, hits = calls["n"], ctx.cache_hits() - hits0
    assert n_grad >= 1
    if model_kind == "vidkl":       # the initial guesses factor; every analytic evaluation after them is a cache hit
        assert hits == n_grad, (hits, n_grad)
    assert x.shape == (D,) and np.all(x >= -2.0) and np.all(x <= 2.0)
    guesses = prng.uniform(key, (8, D), np.float32, np.full(D, -2, np.float32), np.full(D, 2, np.float32))
    best0 = np.max(acq_fn(key, model, guesses, **kw))
    assert acq_fn(key, model, np.asarray(x, np.float64)[None], **kw)[0] >= best0 - 1e-12 * abs(best0)

    # the analytic objective against acq_fn's value and central differences of it, at an interior point
    f = acq._analytic_objective(acq_name, key, model, D, kw)
    x0 = np.array([-0.7, 0.35, 0.4])
    val, grad = f(x0)
    assert np.isclose(val, acq_fn(key, model, x0[None], **kw)[0], rtol=1e-12, atol=0), "value of the gradient path"
    h, fd = 1e-5, np.empty(D)
    for k in range(D):
        e = np.zeros(D)
        e[k] = h
        fd[k] = (acq_fn(key, model, (x0 + e)[None], **kw)[0] - acq_fn(key, model, (x0 - e)[None], **kw)[0]) / (2 * h)
    np.testing.assert_allclose(grad, fd, rtol=1e-5, atol=1e-5 * np.abs(fd).max())


# ------------------------------------------------------------------ refusals, failures, determinism
def raw_call(ctx, kind, X, y, Xn, widths, flats, theta, flags):
    w = np.ascontiguousarray(widths, dtype=np.int64)
    S, P, D = theta.shape[0], Xn.shape[0], X.shape[1]
    outs = [np.empty((S, P)), np.empty((S, P)), np.empty((S, P, D)), np.empty((S, P, D))]
    info = np.zeros(S, dtype=np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    return ctx.lib.b2gp_dkl_posterior_grad(ctx.h, kind, p(X), X.shape[0], D, p(y), 0, p(Xn), P, len(widths), p(w), 0, p(flats), S,
                                           flats.shape[1], p(theta), 0, 1e-6, flags, *(p(o) for o in outs), p(info))


def test_refusals(ctx):
    from gpax_b200 import _ffi
    widths = [16, 2]
    X, y, Xn, flats, theta = problem("RBF", "relu", 50, 3, 4, 1, widths)
    good = _ffi.OUT_MEAN | _ffi.OUT_VAR | _ffi.OUT_DMEAN | _ffi.OUT_DVAR
    assert raw_call(ctx, 0, X, y, Xn, widths, flats, theta, good) == 0
    for kind in (_ffi.KERNEL_NNGP_ERF, _ffi.KERNEL_NNGP_RELU):
        assert raw_call(ctx, kind, X, y, Xn, widths, flats, theta, good) == -1, kind
    for bad in (_ffi.FLAG_F32, _ffi.FLAG_DEVICE_PTRS, _ffi.OUT_COV, _ffi.OUT_SAMPLE):
        assert raw_call(ctx, 0, X, y, Xn, widths, flats, theta, good | bad) == -4, bad


def test_failed_draw_is_nan_and_alone_and_calls_repeat_bit_for_bit(ctx):
    widths = [40, 20, 2]
    X, y, Xn, flats, theta = problem("Matern", "tanh", 200, 17, 300, 4, widths, seed=13)
    theta[2, 2 + 1] = -2.0                            # negative noise: draw 2's k_XX is not positive definite
    out = ctx.dkl_posterior_grad("Matern", X, y, Xn, widths, 1, flats, theta)
    assert out["info"][2] != 0 and all(out["info"][s] == 0 for s in (0, 1, 3))
    for name in ("mean", "var", "dmean", "dvar"):
        assert np.isnan(out[name][2]).all(), name
        assert np.isfinite(out[name][[0, 1, 3]]).all(), name
    good = [0, 1, 3]
    ok = {k: v[good] for k, v in out.items()}
    oracle_check(ok, "Matern", "tanh", X, y, Xn, flats[good], theta[good], widths, False, "draws beside a failed one")
    again = ctx.dkl_posterior_grad("Matern", X, y, Xn, widths, 1, flats, theta)
    for name in ("mean", "var", "dmean", "dvar"):
        np.testing.assert_array_equal(again[name], out[name], err_msg=name)   # NaNs at the same places, equal bits elsewhere
