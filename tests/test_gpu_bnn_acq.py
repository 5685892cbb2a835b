"""Acquisition functions on a BNN, on the GPU.

- b2gp_bnn_predict_grad against the NumPy oracle (the forward pass, then dkl_grad_oracle.input_vjp with a unit
  cotangent) on the fused and the layered route and on a network only the layered route takes; against central
  differences of b2gp_bnn_predict's loc; its loc bit for bit against b2gp_bnn_predict's on the same route;
- launch counts, 70,000 draws, host vs device pointers, determinism, and the refusals made before any launch;
- EI / UCB / POI / UE, Thompson and the q-batch functions on a short NUTS fit against a NumPy restatement from
  BNN.predict's outputs, the KG refusals, and optimize_acq on the closed-form route."""
import ctypes as C

import numpy as np
import pytest

from dkl_grad_oracle import input_vjp
from oracle import acq_oracle as ao
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


def _nets(D, hidden, S, seed):
    """S weight sets of a one-output tanh network: one random network, scaled per draw"""
    rng = np.random.default_rng(seed)
    widths = list(hidden) + [1]
    layers, i = [], D
    for w in widths:
        layers.append((rng.standard_normal((i, w)) / np.sqrt(i), 0.3 * rng.standard_normal(w)))
        i = w
    flats = dko.flatten(layers)[None] * rng.uniform(0.7, 1.3, (S, 1))
    return widths, flats


def _oracle(X, D, widths, flats):
    """(loc [S, P], dloc [S, P, D]) in NumPy"""
    locs, grads = [], []
    for flat in flats:
        layers = dko.unflatten(flat, D, widths)
        H = dko.mlp_forward(X, layers, "tanh")
        locs.append(H[-1][:, 0])
        grads.append(input_vjp(H, layers, "tanh", np.ones((X.shape[0], 1))))
    return np.stack(locs), np.stack(grads)


def _close(got, ref, tol=1e-12):
    np.testing.assert_allclose(got, ref, rtol=0, atol=tol * max(np.abs(ref).max(), 1e-300))


@pytest.mark.parametrize("hidden", [[64, 32], CUSTOM], ids=["default", "custom"])
@pytest.mark.parametrize("D", [1, 3, 64])
@pytest.mark.parametrize("P", [1, 37, 1000])
@pytest.mark.parametrize("S", [1, 7])
def test_predict_grad_matches_oracle_on_both_routes(ctx, S, P, D, hidden):
    rng = np.random.default_rng(S + 10 * P + 100 * D)
    X = rng.uniform(-1.5, 1.5, (P, D))
    widths, flats = _nets(D, hidden, S, seed=P + D)
    rloc, rdloc = _oracle(X, D, widths, flats)
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            loc, dloc = ctx.bnn_predict_grad(X, widths, TANH, flats)
            launches = ctx.last_timing()["launches"]
            ploc, _ = ctx.bnn_predict(X, widths, TANH, flats)
        assert launches == (1 if fused else 3 * len(widths) * S + 1)
        assert loc.shape == (S, P) and dloc.shape == (S, P, D)
        assert np.array_equal(loc, ploc[:, :, 0]), "loc is b2gp_bnn_predict's, bit for bit"
        _close(loc, rloc)
        _close(dloc, rdloc)


def test_network_too_wide_for_shared_memory_takes_the_layered_route(ctx):
    D, P, S = 2, 37, 3
    X = np.random.default_rng(1).uniform(-1, 1, (P, D))
    widths, flats = _nets(D, [512, 512], S, seed=2)
    assert ctx.get_option("bnn_fused") == 1
    loc, dloc = ctx.bnn_predict_grad(X, widths, TANH, flats)
    assert ctx.last_timing()["launches"] == 3 * 3 * S + 1
    ploc, _ = ctx.bnn_predict(X, widths, TANH, flats)
    assert np.array_equal(loc, ploc[:, :, 0])
    rloc, rdloc = _oracle(X, D, widths, flats)
    _close(loc, rloc)
    _close(dloc, rdloc)


@pytest.mark.parametrize("fused", [1, 0])
def test_predict_grad_matches_central_differences_of_predict(ctx, fused):
    D, P, S, h = 3, 9, 4, 1e-5
    X = np.random.default_rng(3).uniform(-1.5, 1.5, (P, D))
    widths, flats = _nets(D, [64, 32], S, seed=4)
    with ctx.options(bnn_fused=fused):
        _, dloc = ctx.bnn_predict_grad(X, widths, TANH, flats)
        fd = np.empty_like(dloc)
        for k in range(D):
            e = np.zeros(D)
            e[k] = h
            up, _ = ctx.bnn_predict(X + e, widths, TANH, flats)
            dn, _ = ctx.bnn_predict(X - e, widths, TANH, flats)
            fd[:, :, k] = (up[:, :, 0] - dn[:, :, 0]) / (2 * h)
    np.testing.assert_allclose(dloc, fd, rtol=1e-6, atol=1e-7 * np.abs(fd).max())


def test_more_draws_than_one_grid_column_holds(ctx):
    """grid.y holds at most 65535 draws, so 70000 draws take two launches of the fused kernel"""
    D, P, S = 2, 5, 70000
    X = np.random.default_rng(5).uniform(-1, 1, (P, D))
    widths, flats = _nets(D, [3], S, seed=5)
    loc, dloc = ctx.bnn_predict_grad(X, widths, TANH, flats)
    assert ctx.last_timing()["launches"] == 2
    rloc, rdloc = _oracle(X, D, widths, flats)
    _close(loc, rloc)
    _close(dloc, rdloc)


def test_device_pointers_and_repeated_calls_give_identical_bits(ctx):
    D, P, S = 4, 70, 9
    X = np.random.default_rng(6).uniform(-1, 1, (P, D))
    widths, flats = _nets(D, [64, 32], S, seed=6)
    for fused in (1, 0):
        with ctx.options(bnn_fused=fused):
            a = ctx.bnn_predict_grad(X, widths, TANH, flats)
            b = ctx.bnn_predict_grad(X, widths, TANH, flats)
            Xd, Pd = ctx.to_device(X), ctx.to_device(flats)
            try:
                c = ctx.bnn_predict_grad(Xd, widths, TANH, Pd)
            finally:
                Xd.free()
                Pd.free()
        for o in (b, c):
            assert np.array_equal(o[0], a[0]) and np.array_equal(o[1], a[1])


def test_refusals_come_before_any_launch(ctx):
    from gpax_b200 import _ffi
    D, P = 2, 4
    X = np.random.default_rng(7).uniform(-1, 1, (P, D))
    widths, flats = _nets(D, [8], 2, seed=7)
    ctx.bnn_predict_grad(X, widths, TANH, flats)
    before = ctx.last_timing()
    w = np.asarray(widths, dtype=np.int64)
    loc, dloc = np.empty((2, P)), np.empty((2, P, D))

    def raw(widths_, S, stride, flags):
        w_ = np.asarray(widths_, dtype=np.int64)
        return ctx.lib.b2gp_bnn_predict_grad(ctx.h, _ffi._ptr(X), P, D, len(w_), _ffi._ptr(w_), TANH, _ffi._ptr(flats), S, stride,
                                             _ffi._ptr(loc), _ffi._ptr(dloc), flags)

    npar = flats.shape[1]
    assert raw(w, 2, npar, _ffi.FLAG_F32) == -4
    assert raw(w, 0, npar, 0) == -1                        # S < 1
    assert raw(w, 2, npar - 1, 0) == -1                    # a stride shorter than one weight set
    two = np.asarray([8, 2], dtype=np.int64)               # two outputs
    assert raw(two, 1, npar, 0) == -1
    with pytest.raises(ValueError):                        # the binding checks the parameter count
        ctx.bnn_predict_grad(X, widths, TANH, flats[:, :-1])
    with pytest.raises(_ffi.B200GPError):
        ctx.bnn_predict_grad(X, [8, 2], TANH, np.zeros((1, _ffi._mlp_nparams(D, np.asarray([8, 2])))))
    assert ctx.last_timing() == before


# ------------------------------------------------------------------ acquisitions on a fitted BNN
def _data(N=48, seed=0):
    rng = np.random.default_rng(seed)
    X = np.sort(rng.uniform(-2, 2, N))
    return X, np.sin(1.5 * X) + 0.05 * rng.standard_normal(N)


@pytest.fixture(scope="module")
def fitted(ctx):
    from gpax_b200 import BNN
    X, y = _data()
    m = BNN(1, 1, hidden_dim=[8, 4], ctx=ctx)
    m.fit(0, X, y, num_warmup=60, num_samples=40, progress_bar=False, print_summary=False)
    return m


ORACLE = {"EI": lambda M, V, kw: ao.ei(M, V, kw.get("best_f"), kw.get("maximize", False)),
          "UCB": lambda M, V, kw: ao.ucb(M, V, kw.get("beta", 0.25), kw.get("maximize", False)),
          "POI": lambda M, V, kw: ao.poi(M, V, kw.get("best_f"), kw.get("xi", 0.01), kw.get("maximize", False)),
          "UE": lambda M, V, kw: ao.ue(M, V)}


@pytest.mark.parametrize("kw", [{}, {"noiseless": True}, {"n": 3, "maximize": True}, {"best_f": 0.2},
                                {"penalty": "inverse_distance", "recent_points": np.array([[0.3], [-1.0]])}],
                         ids=["plain", "noiseless", "n3-max", "best_f", "penalty"])
@pytest.mark.parametrize("name", ["EI", "UCB", "POI", "UE"])
def test_acquisitions_equal_the_restatement_from_predict(fitted, name, kw):
    from gpax_b200 import acquisition as acq
    m = fitted
    X = np.linspace(-2.5, 2.5, 41)[:, None]
    kw = dict(kw)
    if name in ("UCB", "UE"):
        kw.pop("best_f", None)
    if name == "UE":
        kw.pop("maximize", None)
    got = getattr(acq, name)(3, m, X, **kw)
    _, ys = m.predict(3, X, n=kw.get("n", 1), noiseless=kw.get("noiseless", False))
    y = ys[:, :, 0]
    ref = ORACLE[name](y.mean(0), y.var(0), kw)
    if kw.get("penalty"):
        ref = ref - acq.compute_penalty(X, kw["recent_points"], kw["penalty"])
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12 * np.abs(ref).max())
    if kw.get("noiseless"):
        loc, _ = m.predict(3, X, take_point_predictions_mean=False)
        assert np.array_equal(ys, loc)


@pytest.mark.parametrize("n", [1, 4])
def test_thompson_draw_and_shapes(fitted, n):
    from gpax_b200 import acquisition as acq, prng
    m = fitted
    X = np.linspace(-2, 2, 13)
    got = acq.Thompson(9, m, X, n=n)
    S = len(m.get_samples()["noise"])
    idx = prng.randint(prng.as_key(9), (1,), 0, S)
    _, ys = m.predict(9, X, {k: np.asarray(v)[idx] for k, v in m.get_samples().items()}, n)
    assert got.shape == ((1, 1, 13) if n == 1 else (13,))
    assert np.array_equal(got.reshape(-1), ys.reshape(-1))


@pytest.mark.parametrize("name", ["qEI", "qUCB", "qPOI"])
def test_q_batch_rows_equal_the_restatement(fitted, name):
    from gpax_b200 import acquisition as acq
    m = fitted
    X = np.linspace(-2, 2, 17)[:, None]
    got = getattr(acq, name)(4, m, X, subsample_size=5)
    sub = acq._subsample(m.get_samples(), 5, 4)
    loc, _ = bo.predict(X, 1, m.widths, m.to_flat(sub))
    var = np.broadcast_to(sub["noise"][:, None] ** 2, loc.shape[:2])
    base = name[1:]
    ref = np.stack([ORACLE[base](loc[s, :, 0], var[s], {}) for s in range(5)])
    assert got.shape == (5, 17)
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12 * np.abs(ref).max())
    with pytest.raises(ValueError):
        getattr(acq, name)(4, m, X, subsample_size=5, noiseless=True)


def test_kg_and_two_output_bnn_are_refused(fitted, ctx):
    from gpax_b200 import BNN
    from gpax_b200 import acquisition as acq
    X = np.zeros((3, 1))
    for fn in (acq.KG, acq.qKG):
        with pytest.raises(ValueError):
            fn(0, fitted, X)
    two = BNN(1, 2, hidden_dim=[4], ctx=ctx)
    two.fit(0, *_data(24, seed=1), num_warmup=20, num_samples=10, progress_bar=False, print_summary=False)
    for fn in (acq.EI, acq.UCB, acq.POI, acq.UE, acq.Thompson, acq.qEI):
        with pytest.raises(ValueError):
            fn(0, two, X)


@pytest.mark.parametrize("kw", [{}, {"noiseless": True}, {"n": 3}], ids=["plain", "noiseless", "n3"])
@pytest.mark.parametrize("name", ["EI", "UCB", "POI", "UE"])
def test_optimize_acq_takes_the_closed_form_route(fitted, ctx, monkeypatch, name, kw):
    from gpax_b200 import acquisition as acq, prng
    m = fitted
    key = prng.PRNGKey(2)
    original = getattr(acq, name)
    calls = {"acq": 0, "grad": 0}

    def counted(*a, **k):
        calls["acq"] += 1
        return original(*a, **k)
    grad_fn = ctx.bnn_predict_grad

    def counted_grad(*a, **k):
        calls["grad"] += 1
        return grad_fn(*a, **k)
    monkeypatch.setattr(acq, name, counted)
    monkeypatch.setattr(ctx, "bnn_predict_grad", counted_grad)
    assert acq._analytic_kind(counted, m, kw) == name
    x = acq.optimize_acq(key, m, counted, 8, -2.0, 2.0, **kw)
    assert calls["acq"] == 1 and calls["grad"] >= 1, calls
    assert x.shape == () and -2.0 <= float(x) <= 2.0

    # the objective against acq_fn's value and central differences of it, at an interior point
    with acq._bnn_objective(name, key, m, 1, kw) as f:
        for x0 in (np.array([-0.6]), np.array([0.45])):
            val, grad = f(x0)
            ref = original(key, m, x0[None], **kw)[0]
            assert abs(val - ref) <= 1e-12 * max(abs(ref), 1e-300), (val, ref)
            h = 1e-5
            fd = (original(key, m, (x0 + h)[None], **kw)[0] - original(key, m, (x0 - h)[None], **kw)[0]) / (2 * h)
            assert abs(grad[0] - fd) <= 1e-6 * max(abs(fd), 1e-3), (grad, fd)
