"""b2gp_bnn_loglik_draws on the GPU: every draw bit for bit against its own b2gp_bnn_loglik call on the fused and the
layered route, the NumPy oracle (oracle/bnn_oracle.py), chunks of more than 65535 draws, launch counts, determinism,
refusals before any launch, BNNLogJoint.batch against __call__, and vectorized BNN chains against sequential ones."""
import ctypes as C

import numpy as np
import pytest

from oracle import bnn_oracle as bo
from oracle import dkl_oracle as dko

pytestmark = pytest.mark.gpu

TANH = 1
HIDDEN = {"default": [64, 32], "custom": [16, 8, 4]}


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def _problem(N, D, hidden, O, S, seed, pad=3):
    """X [N, D], y [N, O], widths, S weight sets as a strided view (row stride nparams + pad) and S noise scales"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1.5, 1.5, (N, D))
    y = np.sin(2 * X[:, :1]) + 0.3 * np.arange(O)[None, :] + 0.1 * rng.standard_normal((N, O))
    widths = list(hidden) + [O]
    sets = []
    for _ in range(S):
        layers, i = [], D
        for w in widths:
            layers.append((rng.standard_normal((i, w)) / np.sqrt(i), 0.3 * rng.standard_normal(w)))
            i = w
        sets.append(dko.flatten(layers))
    P = sets[0].size
    buf = np.full((S, P + pad), np.nan)
    buf[:, :P] = np.stack(sets)
    return X, y, widths, buf[:, :P], rng.uniform(0.05, 0.8, S)


def _same(a, b):
    return a[0] == b[0] and a[1] == b[1] and np.array_equal(a[2], b[2])


def _check_draws(ctx, X, y, widths, params, sigma):
    """draws call vs one bnn_loglik per draw on the same inputs (host or device): identical bits"""
    vals, gs, gp = ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma)
    for s in range(params.shape[0]):
        one = ctx.bnn_loglik(X, y, widths, TANH, np.ascontiguousarray(params[s]), sigma[s])
        assert _same((vals[s], gs[s], gp[s]), one), f"draw {s}"
    return vals, gs, gp


@pytest.mark.parametrize("hidden", list(HIDDEN))
@pytest.mark.parametrize("S", [1, 3, 8])
@pytest.mark.parametrize("N", [1, 31, 32, 33, 257, 20000])
def test_draws_match_single_calls_bit_for_bit(ctx, N, S, hidden):
    """N = 20000 is 625 row tiles, more than the fused grid's width on an H100, so the tile loop strides"""
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            for D, O in ((1, 1), (5, 2)):
                X, y, widths, params, sigma = _problem(N, D, HIDDEN[hidden], O, S, seed=N + S + D)
                assert params.strides[0] > 8 * params.shape[1]
                _check_draws(ctx, X, y, widths, params, sigma)
                Xd, yd = ctx.to_device(X), ctx.to_device(y)
                try:
                    _check_draws(ctx, Xd, yd, widths, params, sigma)
                finally:
                    Xd.free()
                    yd.free()


@pytest.mark.parametrize("hidden", list(HIDDEN))
def test_draws_match_the_oracle_on_both_routes(ctx, hidden):
    X, y, widths, params, sigma = _problem(1000, 3, HIDDEN[hidden], 2, 4, seed=9)
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            vals, gs, gp = ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma)
        for s in range(4):
            rv, rgs, rgp, scale = bo.loglik(X, y, 3, widths, params[s], sigma[s])
            rtol = 1e-11                          # test_gpu_bnn.py's tolerance for b2gp_bnn_loglik
            assert abs(vals[s] - rv) <= rtol * (abs(rv) + 1.0)
            assert abs(gs[s] - rgs) <= rtol * (abs(rgs) + 1.0)
            assert np.all(np.abs(gp[s] - rgp) <= rtol * (scale + 1e-3 * scale.max()))


def test_more_draws_than_one_grid_column_holds(ctx):
    """grid.y holds at most 65535 draws: 70000 draws of a tiny network take two chunks, two launches each"""
    S = 70000
    X, y, widths, params, _ = _problem(5, 1, [3], 1, 1, seed=4)
    rng = np.random.default_rng(5)
    params = params[0][None] * rng.uniform(0.5, 1.5, (S, 1))
    sigma = rng.uniform(0.05, 0.5, S)
    vals, gs, gp = ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma)
    assert ctx.last_timing()["launches"] == 4
    for s in (0, 65534, 65535, S - 1):
        assert _same((vals[s], gs[s], gp[s]), ctx.bnn_loglik(X, y, widths, TANH, params[s], sigma[s])), s


@pytest.mark.parametrize("S", [1, 5, 40])
def test_launches_per_call(ctx, S):
    X, y, widths, params, sigma = _problem(300, 1, [64, 32], 1, S, seed=S)
    ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma)
    assert ctx.last_timing()["launches"] == 2
    with ctx.options(bnn_fused=0):
        ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma)
        assert ctx.last_timing()["launches"] == S * (9 * len(widths) - 1)


def test_repeated_calls_give_identical_bits(ctx):
    X, y, widths, params, sigma = _problem(4099, 2, [64, 32], 2, 6, seed=2)
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            a = ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma)
            b = ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma)
        assert all(np.array_equal(u, v) for u, v in zip(a, b))


def test_without_params_gradient(ctx):
    X, y, widths, params, sigma = _problem(100, 1, [16, 8, 4], 1, 3, seed=6)
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            full = ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma)
            part = ctx.bnn_loglik_draws(X, y, widths, TANH, params, sigma, want_params=False)
        assert part[2] is None and np.array_equal(part[0], full[0]) and np.array_equal(part[1], full[1])


def test_refusals_before_any_launch(ctx):
    from gpax_b200 import _ffi
    S = 3
    X, y, widths, params, sigma = _problem(40, 1, [8], 1, S, seed=1)
    w = np.asarray(widths, dtype=np.int64)
    P = params.shape[1]
    flat = np.ascontiguousarray(params)
    p = _ffi._ptr

    def call(X=X, y=y, w=w, params=flat, stride=P, sigma=sigma, flags=0, S=S, value=True, gsig=True, nw=len(widths)):
        val, gs, gp = np.full(S if S > 0 else 1, 7.0), np.full(S if S > 0 else 1, 7.0), np.full((max(S, 1), P), 7.0)
        rc = ctx.lib.b2gp_bnn_loglik_draws(ctx.h, p(X), 40, 1, p(y), 1, nw, p(w), TANH, S, p(params), stride, p(sigma),
                                           flags, p(val) if value else None, p(gs) if gsig else None, p(gp))
        return rc, val, gs, gp

    rc, *good = call()
    assert rc == 0
    before = ctx.last_timing()
    cases = []
    for bad in (0.0, -0.1, np.inf, np.nan):
        sg = sigma.copy()
        sg[2] = bad
        cases.append(dict(sigma=sg))
    cases += [dict(flags=_ffi.FLAG_F32), dict(stride=P - 1), dict(stride=-1), dict(S=0), dict(X=None), dict(y=None),
              dict(params=None), dict(sigma=None), dict(value=False), dict(gsig=False), dict(w=None), dict(nw=0)]
    for kw in cases:
        rc, val, gs, gp = call(**kw)
        assert rc != 0, kw
        assert (val == 7.0).all() and (gs == 7.0).all() and (gp == 7.0).all(), kw
        assert ctx.last_timing() == before, kw             # no call began: the last call's timing is untouched
    assert ctx.get_option("bnn_fused") == 1
    rc, *again = call()
    assert rc == 0 and all(np.array_equal(a, b) for a, b in zip(good, again))
    with pytest.raises(_ffi.B200GPError):
        ctx.bnn_loglik_draws(X, y, widths, TANH, params, [0.1, -0.1, 0.1])


# ------------------------------------------------------------------------------------------------ BNN end to end
def test_log_joint_batch_rows_equal_single_calls(ctx):
    from gpax_b200 import BNN
    from gpax_b200.bnn import BNNLogJoint
    rng = np.random.default_rng(7)
    X = rng.uniform(-2, 2, (50, 1))
    y = np.sin(1.5 * X) + 0.05 * rng.standard_normal((50, 1))
    m = BNN(1, 1, ctx=ctx)
    lj = BNNLogJoint(m, X, y, rng)
    try:
        u0 = lj.init_u()
        U = u0[None] + 0.1 * rng.standard_normal((5, u0.size))
        U[1, 0] = 1e6                                     # the noise overflows: -inf without a library call
        U[3, 0] = np.nan
        for fused in (1, 0):
            with ctx.options(bnn_fused=fused):
                for jac in (False, True):
                    vals, grads = lj.batch(U, jac)
                    for r in range(len(U)):
                        v, g = lj(U[r], jac)
                        assert vals[r] == v and np.array_equal(grads[r], g), (fused, jac, r)
        assert vals[1] == -np.inf and vals[3] == -np.inf and np.isfinite(vals[[0, 2, 4]]).all()
    finally:
        lj.close()


def test_vectorized_fit_matches_sequential(ctx):
    from gpax_b200 import BNN
    rng = np.random.default_rng(0)
    X = np.sort(rng.uniform(-2, 2, 40))
    y = np.sin(1.5 * X) + 0.05 * rng.standard_normal(40)
    runs = {}
    for method in ("sequential", "vectorized"):
        m = BNN(1, 1, hidden_dim=[8, 4], ctx=ctx)
        calls = {"bnn_loglik": 0, "bnn_loglik_draws": 0}
        for k in calls:
            def wrap(*a, _f=getattr(ctx, k), _k=k, **kw):
                calls[_k] += 1
                return _f(*a, **kw)
            setattr(ctx, k, wrap)
        try:
            m.fit(0, X, y, num_warmup=20, num_samples=15, num_chains=3, chain_method=method, progress_bar=False,
                  print_summary=False)
        finally:
            for k in calls:
                delattr(ctx, k)
        runs[method] = (m.get_samples(chain_dim=True), m.mcmc.stats, calls)
    (s_seq, st_seq, c_seq), (s_vec, st_vec, c_vec) = runs["sequential"], runs["vectorized"]
    assert list(s_seq) == list(s_vec)
    for k in s_seq:
        assert s_seq[k].shape[:2] == (3, 15) and np.array_equal(s_seq[k], s_vec[k]), k
    assert st_seq == st_vec
    rounds = max(np.diff([0] + [s["grad_evals"] for s in st_vec]))
    assert c_vec == {"bnn_loglik": 0, "bnn_loglik_draws": rounds}
    assert c_seq["bnn_loglik_draws"] == 0 and c_seq["bnn_loglik"] == st_seq[-1]["grad_evals"]
