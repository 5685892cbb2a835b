"""The fully Bayesian MLP on the GPU: b2gp_bnn_loglik and b2gp_bnn_predict against the NumPy oracle (oracle/bnn_oracle.py)
on the fused and the layered route, the route witness (launch counts), determinism, host vs device pointers, and BNN end
to end."""
import numpy as np
import pytest

from oracle import bnn_oracle as bo
from oracle import dkl_oracle as dko

pytestmark = pytest.mark.gpu

TANH = 1
CUSTOM = [16, 8, 4]


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def _net(D, hidden, O, seed):
    rng = np.random.default_rng(seed)
    widths = list(hidden) + [O]
    layers, i = [], D
    for w in widths:
        layers.append((rng.standard_normal((i, w)) / np.sqrt(i), 0.3 * rng.standard_normal(w)))
        i = w
    return widths, dko.flatten(layers)


def _problem(N, D, hidden, O, seed):
    rng = np.random.default_rng(seed + 1)
    X = rng.uniform(-1.5, 1.5, (N, D))
    y = np.sin(2 * X[:, :1]) + 0.3 * np.arange(O)[None, :] + 0.1 * rng.standard_normal((N, O))
    widths, flat = _net(D, hidden, O, seed)
    return X, y, widths, flat


def _check_loglik(got, ref, rtol):
    val, gs, gp = got
    rv, rgs, rgp, scale = ref
    n = scale.size
    assert abs(val - rv) <= rtol * (abs(rv) + 1.0), (val, rv)
    assert abs(gs - rgs) <= rtol * (abs(rgs) + 1.0), (gs, rgs)
    err = np.abs(gp - rgp)
    bound = rtol * (scale + 1e-3 * scale.max())
    assert np.all(err <= bound), f"grad_params: worst {np.max(err / bound):.3g} x the bound over {n} entries"


@pytest.mark.parametrize("hidden", [[64, 32], CUSTOM], ids=["default", "custom"])
@pytest.mark.parametrize("D,O", [(1, 1), (3, 3), (64, 1)])
@pytest.mark.parametrize("N", [1, 37, 1000, 5000])
def test_loglik_matches_oracle_on_both_routes(ctx, N, D, O, hidden):
    X, y, widths, flat = _problem(N, D, hidden, O, seed=N + 7 * D + O)
    sigma = 0.3
    ref = bo.loglik(X, y, D, widths, flat, sigma)
    out = {}
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            out[fused] = ctx.bnn_loglik(X, y, widths, TANH, flat, sigma)
            launches = ctx.last_timing()["launches"]
        _check_loglik(out[fused], ref, 1e-11)
        assert launches == (2 if fused else 9 * len(widths) - 1)
    # the two routes against each other
    _check_loglik(out[1], (out[0][0], out[0][1], out[0][2], ref[3]), 1e-12)


def test_route_rule_takes_layered_for_wide_networks(ctx):
    X, y, widths, flat = _problem(300, 1, [512, 512], 1, seed=3)
    assert ctx.get_option("bnn_fused") == 1
    got = ctx.bnn_loglik(X, y, widths, TANH, flat, 0.2)
    assert ctx.last_timing()["launches"] == 9 * 3 - 1
    _check_loglik(got, bo.loglik(X, y, 1, widths, flat, 0.2), 1e-11)
    loc, _ = ctx.bnn_predict(X, widths, TANH, np.stack([flat, 0.9 * flat]))
    assert ctx.last_timing()["launches"] == 2 * (3 * 3 + 1)
    ref, _ = bo.predict(X, 1, widths, np.stack([flat, 0.9 * flat]))
    np.testing.assert_allclose(loc, ref, rtol=0, atol=1e-12 * np.abs(ref).max())


def test_default_network_takes_the_fused_route_at_the_largest_supported_shape(ctx):
    X, y, widths, flat = _problem(100, 64, [64, 32], 8, seed=5)
    ctx.bnn_loglik(X, y, widths, TANH, flat, 0.5)
    assert ctx.last_timing()["launches"] == 2
    ctx.bnn_predict(X, widths, TANH, flat)
    assert ctx.last_timing()["launches"] == 1


def test_loglik_deterministic_and_device_pointers_give_the_same_bits(ctx):
    X, y, widths, flat = _problem(4099, 3, [64, 32], 2, seed=11)
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            a = ctx.bnn_loglik(X, y, widths, TANH, flat, 0.25)
            b = ctx.bnn_loglik(X, y, widths, TANH, flat, 0.25)
            Xd, yd = ctx.to_device(X), ctx.to_device(y)
            try:
                c = ctx.bnn_loglik(Xd, yd, widths, TANH, flat, 0.25)
            finally:
                Xd.free()
                yd.free()
        for o in (b, c):
            assert o[0] == a[0] and o[1] == a[1] and np.array_equal(o[2], a[2])


def test_fp32_io_is_refused(ctx):
    from gpax_b200 import _ffi
    import ctypes as C
    X, y, widths, flat = _problem(10, 1, [8], 1, seed=1)
    w = np.asarray(widths, dtype=np.int64)
    v, g = C.c_double(), C.c_double()
    rc = ctx.lib.b2gp_bnn_loglik(ctx.h, _ffi._ptr(X), 10, 1, _ffi._ptr(y), 1, len(widths), _ffi._ptr(w), TANH, _ffi._ptr(flat),
                                 0.1, _ffi.FLAG_F32, C.byref(v), C.byref(g), None)
    assert rc != 0


def test_sigma_must_be_positive_and_finite(ctx):
    from gpax_b200 import _ffi
    X, y, widths, flat = _problem(10, 1, [8], 1, seed=1)
    for bad in (0.0, -0.1, np.inf, np.nan):
        with pytest.raises(_ffi.B200GPError):
            ctx.bnn_loglik(X, y, widths, TANH, flat, bad)


def test_predict_more_draws_than_one_grid_column_holds(ctx):
    """grid.y holds at most 65535 draws, so 70000 draws take two launches of the fused kernel"""
    D, O, Pn, S = 1, 1, 5, 70000
    rng = np.random.default_rng(4)
    X = rng.uniform(-1, 1, (Pn, D))
    widths, flat = _net(D, [3], O, seed=4)
    flats = flat[None] * rng.uniform(0.5, 1.5, (S, 1))
    sigma = rng.uniform(0.05, 0.5, S)
    eps = rng.standard_normal((S, 1, Pn, O))
    loc, ys = ctx.bnn_predict(X, widths, TANH, flats, sigma, eps)
    assert ctx.last_timing()["launches"] == 2
    rloc, rys = bo.predict(X, D, widths, flats, sigma, eps)
    np.testing.assert_allclose(loc, rloc, rtol=0, atol=1e-12 * np.abs(rloc).max())
    np.testing.assert_allclose(ys, rys, rtol=0, atol=1e-12 * np.abs(rys).max())


@pytest.mark.parametrize("hidden", [[64, 32], CUSTOM], ids=["default", "custom"])
@pytest.mark.parametrize("S", [1, 7, 300])
@pytest.mark.parametrize("n", [1, 4])
def test_predict_matches_oracle_on_both_routes(ctx, S, n, hidden):
    D, O, Pn = 2, 3, 129
    rng = np.random.default_rng(S * 10 + n)
    X = rng.uniform(-1.5, 1.5, (Pn, D))
    widths, flat = _net(D, hidden, O, seed=S)
    flats = flat[None] * rng.uniform(0.7, 1.3, (S, 1))
    sigma = rng.uniform(0.05, 0.5, S)
    eps = rng.standard_normal((S, n, Pn, O))
    rloc, rys = bo.predict(X, D, widths, flats, sigma, eps)
    out = {}
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            out[fused] = ctx.bnn_predict(X, widths, TANH, flats, sigma, eps)
            launches = ctx.last_timing()["launches"]
        assert launches == (1 if fused else S * (3 * len(widths) + 1))
        np.testing.assert_allclose(out[fused][0], rloc, rtol=0, atol=1e-12 * np.abs(rloc).max())
        np.testing.assert_allclose(out[fused][1], rys, rtol=0, atol=1e-12 * np.abs(rys).max())
    np.testing.assert_allclose(out[1][1], out[0][1], rtol=0, atol=1e-12 * np.abs(rys).max())


# ------------------------------------------------------------------------------------------------ BNN end to end
def _data(N=64, seed=0):
    rng = np.random.default_rng(seed)
    X = np.sort(rng.uniform(-2, 2, N))
    f = np.sin(1.5 * X)
    return X, f, f + 0.05 * rng.standard_normal(N)


@pytest.fixture(scope="module")
def fitted(ctx):
    from gpax_b200 import BNN
    X, f, y = _data()
    m = BNN(1, 1, hidden_dim=[8, 4], ctx=ctx)
    m.fit(0, X, y, num_warmup=100, num_samples=100, progress_bar=False, print_summary=False)
    return m, X, f, y


def test_bnn_sites_and_mu(fitted):
    m, X, _, _ = fitted
    s = m.get_samples()
    shapes = {"w0": (100, 1, 8), "b0": (100, 8), "w1": (100, 8, 4), "b1": (100, 4), "w2": (100, 4, 1), "b2": (100, 1),
              "noise": (100,), "mu": (100, 64, 1)}
    assert {k: v.shape for k, v in s.items()} == shapes
    sc = m.get_samples(chain_dim=True)
    assert {k: v.shape for k, v in sc.items()} == {k: (1,) + v for k, v in shapes.items()}
    ref, _ = bo.predict(X[:, None], 1, [8, 4, 1], m.to_flat(s))
    np.testing.assert_allclose(s["mu"], ref, rtol=0, atol=1e-12 * np.abs(ref).max())
    means = m.get_param_means()
    assert isinstance(means["noise"], float) and means["w1"].shape == (8, 4) and "mu" not in means


def test_bnn_predict_shapes_and_fit_quality(fitted):
    m, X, f, _ = fitted
    mean, ys = m.predict(1, X, n=3)
    assert mean.shape == (64, 1) and ys.shape == (100, 64, 1)
    loc, ys2 = m.predict(1, X, n=3, take_point_predictions_mean=False)
    assert loc.shape == (100, 64, 1) and np.array_equal(ys, ys2)
    # the posterior predictive mean follows the noiseless targets (noise sd 0.05 on sin(1.5 x), |f| <= 1)
    rmse = float(np.sqrt(np.mean((mean[:, 0] - f) ** 2)))
    assert rmse < 0.15, rmse
    loc1, s1 = m.sample_single_posterior_predictive(2, X[:5], {k: v[0] for k, v in m.get_samples().items()}, 4)
    assert loc1.shape == (5, 1) and s1.shape == (5, 1)


def test_bnn_filter_nans(fitted):
    m, X, _, _ = fitted
    s = {k: v[:5].copy() for k, v in m.get_samples().items()}
    s["w2"][2] = np.nan
    _, ys = m.predict(0, X, samples=s, filter_nans=True)
    assert ys.shape == (4, 64, 1) and np.isfinite(ys).all()


def test_bnn_noise_prior_dist_and_prior_samples(ctx):
    from gpax_b200 import BNN
    from gpax_b200 import priors as P
    X, _, y = _data(32, seed=1)
    m = BNN(1, 1, noise_prior_dist=P.LogNormal(-4.0, 0.05), hidden_dim=[4], ctx=ctx)
    m.fit(0, X, y, num_warmup=60, num_samples=40, progress_bar=False, print_summary=False)
    noise = m.get_samples()["noise"]
    assert np.all((noise > np.exp(-4.3)) & (noise < np.exp(-3.7)))      # a tight prior dominates
    ys = m.sample_from_prior(0, X, num_samples=6)
    assert ys.shape == (6, 32, 1) and np.isfinite(ys).all()


def test_bnn_default_architecture_short_fit(ctx):
    """the fused likelihood inside NUTS with the default [64, 32] network"""
    from gpax_b200 import BNN
    X, f, y = _data(48, seed=2)
    m = BNN(1, 1, ctx=ctx)
    m.fit(0, X, y, num_warmup=30, num_samples=20, progress_bar=False, print_summary=False)
    assert m.get_samples()["w1"].shape == (20, 64, 32)
    assert m.mcmc.stats[0]["grad_evals"] > 50
    mean, _ = m.predict(0, X)
    assert mean.shape == (48, 1) and np.isfinite(mean).all()
