"""GPU: b2gp_mll_draws, S likelihoods on one X in lock-step groups, and NUTS fits whose chains run under
chain_method="vectorized".

Draw s of ctx.mll_draws must be ctx.mll(theta[s], yres[s]) bit for bit on every route and however the draws are grouped:
that is what keeps vectorized chains identical to sequential ones."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KINDS = ["RBF", "Matern", "Periodic", "NNGP_erf", "NNGP_relu"]


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
    if kind.startswith("NNGP"):     # (depth, unused, var_w, noise, var_b)
        theta = np.column_stack([np.full(S, 2.0), np.zeros((S, d - 1)), rng.uniform(0.8, 1.5, S), rng.uniform(0.02, 0.1, S),
                                 rng.uniform(0.05, 0.3, S)])
    else:
        theta = np.column_stack([rng.uniform(0.2, 0.5, (S, d)), rng.uniform(0.7, 1.3, S), rng.uniform(0.02, 0.1, S),
                                 rng.uniform(0.6, 1.2, S)])
    return X, Y, theta


def same(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def check_bits(ctx, kind, X, Y, theta, shared):
    """mll_draws against one ctx.mll per draw: value, gradient, alpha and info bit for bit"""
    yres = Y[0] if shared else Y
    val, grad, alpha, info = ctx.mll_draws(kind, X, yres, theta, want_grad=True, want_alpha=True)
    for s in range(theta.shape[0]):
        v, g, a, i = ctx.mll(kind, X, Y[0] if shared else Y[s], theta[s], want_grad=True, want_alpha=True)
        assert info[s] == i
        assert same(np.array(val[s]), np.array(v)), (s, val[s], v)
        assert same(grad[s], g), s
        if i == 0:
            assert same(alpha[s], a), s
    return val, grad, alpha, info


def counted(ctx, fn):
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("N", [1, 17, 128, 129, 700])
def test_draws_match_mll_bit_for_bit(ctx, kind, N):
    for S in (1, 3, 8):
        X, Y, theta = inputs(kind, N, S)
        for shared in (True, False):
            _, info = check_bits(ctx, kind, X, Y, theta, shared)[::3]
            assert (info == 0).all()


@pytest.mark.parametrize("kind", ["RBF", "Periodic", "NNGP_relu"])
def test_tall_fp64_route(ctx, kind):
    X, Y, theta = inputs(kind, 700, 3)
    with ctx.options(tall_min_fp64=256, panel=256):
        _, moved = counted(ctx, lambda: check_bits(ctx, kind, X, Y, theta, False))
    # the tall route was taken by the three draws of mll_draws and the three ctx.mll references
    assert moved["potrf_tall_fp64"] == 6 and moved["mll_draws_batch"] == 1


@pytest.mark.parametrize("kind", ["RBF", "NNGP_erf"])
def test_int8_route_runs_per_draw(ctx, kind):
    X, Y, theta = inputs(kind, 700, 3)
    with ctx.options(ozaki=7, tall_min=512):
        _, moved = counted(ctx, lambda: check_bits(ctx, kind, X, Y, theta, True))
    assert moved["mll_draws_batch"] == 3 and moved["potrf_tall"] == 6


def test_group_split_keeps_the_bits(ctx):
    X, Y, theta = inputs("Matern", 300, 8)
    ref = ctx.mll_draws("Matern", X, Y, theta, want_alpha=True)
    for B, groups in ((1, 8), (3, 3), (8, 1)):
        with ctx.options(draw_batch=B):
            got, moved = counted(ctx, lambda: check_bits(ctx, "Matern", X, Y, theta, False))
        assert moved["mll_draws_batch"] == groups
        for a, b in zip(got, ref):
            assert same(a, b)


@pytest.mark.parametrize("kind", ["RBF", "NNGP_erf"])
def test_launches_do_not_grow_with_draws(ctx, kind):
    X, Y, theta = inputs(kind, 129, 8)
    ctx.mll(kind, X, Y[0], theta[0], want_grad=True)
    one_mll = ctx.last_timing()["launches"]
    ctx.mll_draws(kind, X, Y[0], theta[:1])
    one = ctx.last_timing()["launches"]
    _, moved = counted(ctx, lambda: ctx.mll_draws(kind, X, Y[0], theta))
    eight = ctx.last_timing()["launches"]
    assert eight == one and moved["mll_draws_batch"] == 1
    # a group of one is ctx.mll's sequence plus the copies of theta and y into the draw region, the zeroing of K^{-1}
    # (a memset in ctx.mll) and the copy of the results out
    assert one == one_mll + 4
    ctx.mll(kind, X, Y[0], theta[0], want_grad=True)
    assert ctx.last_timing()["launches"] == one_mll


def test_failed_draw_is_isolated_and_calls_repeat(ctx):
    X, Y, theta = inputs("RBF", 129, 4)
    theta[2, 3] = -0.5                       # noise -0.5 + jitter: K is not positive definite
    val, grad, alpha, info = check_bits(ctx, "RBF", X, Y, theta, False)
    assert info[2] != 0 and np.isnan(val[2]) and np.isnan(grad[2]).all() and np.isnan(alpha[2]).all()
    assert (info[[0, 1, 3]] == 0).all() and np.isfinite(val[[0, 1, 3]]).all()
    again = ctx.mll_draws("RBF", X, Y, theta, want_alpha=True)
    for a, b in zip(again, (val, grad, alpha, info)):
        assert same(a, b)


def test_refusals_before_any_launch(ctx):
    from gpax_b200 import _ffi
    X, Y, theta = inputs("RBF", 64, 2)
    val, info = np.zeros(2), np.zeros(2, dtype=np.int32)
    p = lambda a: C.c_void_p(a.ctypes.data)     # noqa: E731
    for flags in (_ffi.FLAG_F32, _ffi.FLAG_DEVICE_PTRS):
        before = ctx.path_counts()
        rc = ctx.lib.b2gp_mll_draws(ctx.h, _ffi.KERNEL_RBF, p(X), 64, p(Y), 64, 2, 2, p(theta), 1e-6, flags, p(val), None, None,
                                    p(info))
        assert rc == -4 and ctx.path_counts() == before
    with pytest.raises(ValueError):
        ctx.mll_draws("RBF", X, Y[:, :10], theta)
    with pytest.raises(_ffi.B200GPError):      # NNGP depth checked per draw, before any launch
        bad = inputs("NNGP_erf", 64, 2)[2]
        bad[1, 0] = 1.5
        ctx.mll_draws("NNGP_erf", X, Y[0], bad)


# ---------------------------------------------------------------------------------------------- fits
def _mean_fn(x, params):
    return params["a"] * x ** params["b"]


def _mean_fn_priors():
    from gpax_b200 import priors as numpyro
    return {"a": numpyro.sample("a", numpyro.distributions.LogNormal(0, 1)),
            "b": numpyro.sample("b", numpyro.distributions.Normal(3, 1))}


def _data(n=12, seed=0):
    rng = np.random.default_rng(seed)
    X = np.linspace(1, 2, n) + 0.05 * rng.standard_normal(n)
    return X, 10 * X ** 2 + 0.1 * rng.standard_normal(n)


def _model(name, ctx):
    import gpax_b200
    X, y = _data()
    if name in ("RBF", "Periodic"):
        return gpax_b200.ExactGP(1, name, ctx=ctx), (X, y), "mll_draws"
    if name in ("erf", "relu"):
        return gpax_b200.iBNN(1, depth=2, activation=name, ctx=ctx), ((X - 1.5) * 2, y / 40), "mll_draws"
    if name == "mean_fn_prior":
        return gpax_b200.ExactGP(1, "RBF", mean_fn=_mean_fn, mean_fn_prior=_mean_fn_priors, ctx=ctx), (X, y), "mll_draws"
    if name == "vExactGP":
        Xb = np.stack([_data(8, s)[0] for s in range(3)])
        return gpax_b200.vExactGP(1, "RBF", ctx=ctx), (Xb, 10 * Xb ** 2), "mll_batch"
    if name == "UIGP":
        Xu = (X - 1) / 1.0
        return gpax_b200.UIGP(1, "RBF", ctx=ctx), (Xu, np.sin(3 * Xu)), "mll_batch"
    if name == "MeasuredNoiseGP":
        return gpax_b200.MeasuredNoiseGP(1, "RBF", ctx=ctx), (X, y, np.full(X.size, 0.05)), None
    raise KeyError(name)


@pytest.mark.parametrize("name", ["RBF", "Periodic", "erf", "relu", "mean_fn_prior", "vExactGP", "UIGP", "MeasuredNoiseGP"])
def test_vectorized_fit_matches_sequential(ctx, name):
    runs = {}
    for method in ("sequential", "vectorized"):
        m, args, call = _model(name, ctx)
        calls = {"mll": 0, "mll_draws": 0, "mll_batch": 0}
        for k in calls:
            def wrap(*a, _f=getattr(ctx, k), _k=k, **kw):
                calls[_k] += 1
                return _f(*a, **kw)
            setattr(ctx, k, wrap)
        try:
            m.fit(0, *args, num_warmup=30, num_samples=30, num_chains=3, chain_method=method, progress_bar=False,
                  print_summary=False)
        finally:
            for k in calls:
                delattr(ctx, k)
        runs[method] = (m.mcmc.get_samples(group_by_chain=True), m.mcmc.stats, calls)
    (s_seq, st_seq, c_seq), (s_vec, st_vec, c_vec) = runs["sequential"], runs["vectorized"]
    assert sorted(s_seq) == sorted(s_vec)
    for k in s_seq:
        assert s_seq[k].shape[:2] == (3, 30) and same(np.asarray(s_seq[k]), np.asarray(s_vec[k])), k
    assert st_seq == st_vec
    _, _, call = _model(name, ctx)
    if call is not None:
        # one likelihood call per round: rounds = the longest chain's evaluations
        own = np.diff([0] + [s["grad_evals"] for s in st_vec])
        assert c_vec[call] == max(own)
        if call == "mll_draws":
            assert c_vec["mll"] == 0 and c_seq["mll_draws"] == 0
