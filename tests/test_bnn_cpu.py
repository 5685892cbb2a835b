"""BNN on the CPU: the oracle's analytic gradient against central differences, the flat <-> site-dict layout, _set_data,
the refusals, BNNLogJoint's prior and Jacobian terms against finite differences (a stub stands in for the context's
likelihood), and predict's random stream (prng)."""
import numpy as np
import pytest

from oracle import bnn_oracle as bo


def _flat(D, widths, seed):
    rng = np.random.default_rng(seed)
    n = sum(i * w + w for i, w in zip([D] + widths[:-1], widths))
    return 0.5 * rng.standard_normal(n)


@pytest.mark.parametrize("D,widths", [(1, [6, 4, 1]), (3, [5, 2])])
def test_oracle_gradient_against_central_differences(D, widths):
    rng = np.random.default_rng(1)
    X = rng.uniform(-1, 1, (9, D))
    y = rng.standard_normal((9, widths[-1]))
    flat, sigma = _flat(D, widths, 2), 0.4
    _, gs, gp, _ = bo.loglik(X, y, D, widths, flat, sigma)
    h = 1e-6
    num = np.array([(bo.loglik(X, y, D, widths, flat + h * e, sigma)[0] - bo.loglik(X, y, D, widths, flat - h * e, sigma)[0]) / (2 * h)
                    for e in np.eye(flat.size)])
    np.testing.assert_allclose(gp, num, rtol=1e-6, atol=1e-6 * np.abs(num).max())
    ns = (bo.loglik(X, y, D, widths, flat, sigma + h)[0] - bo.loglik(X, y, D, widths, flat, sigma - h)[0]) / (2 * h)
    assert abs(gs - ns) <= 1e-6 * abs(ns)


def test_flat_layout_round_trip():
    from gpax_b200 import BNN
    m = BNN(3, 2, hidden_dim=[4, 5])
    assert m.widths == [4, 5, 2] and m.site_names() == ["w0", "b0", "w1", "b1", "w2", "b2", "noise"]
    flat = np.arange(3 * 4 + 4 + 4 * 5 + 5 + 5 * 2 + 2, dtype=np.float64)
    d = m.from_flat(flat)
    assert d["w0"].shape == (3, 4) and d["b2"].shape == (2,)
    assert np.array_equal(d["w0"].ravel(), flat[:12]) and np.array_equal(d["b0"], flat[12:16])
    assert np.array_equal(m.to_flat(d), flat)
    batch = m.from_flat(np.stack([flat, 2 * flat]))
    assert batch["w1"].shape == (2, 4, 5) and np.array_equal(m.to_flat(batch)[1], 2 * flat)
    assert np.array_equal(m._weight_mask(), np.r_[np.ones(12), np.zeros(4), np.ones(20), np.zeros(5), np.ones(10), np.zeros(2)] > 0)


def test_set_data_and_default_architecture():
    from gpax_b200 import BNN
    m = BNN(1, 1)
    assert m.hidden_dim == [64, 32]
    X, y = m._set_data(np.ones(5), np.ones(5))
    assert X.shape == (5, 1) and y.shape == (5, 1) and m._set_data(np.ones(5)).shape == (5, 1)
    X, y = BNN(2, 3)._set_data(np.ones((5, 2)), np.ones((5, 3)))
    assert X.shape == (5, 2) and y.shape == (5, 3)


def test_shapes_that_do_not_match_the_network_are_refused():
    """a wrong input width or output count is a ValueError before anything reaches the library (the flat parameter
    vector is sized from input_dim, the library would size it from X)"""
    from gpax_b200 import BNN
    m = BNN(1, 2, hidden_dim=[3], ctx=_StubCtx())
    with pytest.raises(ValueError):
        m.fit(0, np.ones((5, 2)), np.ones((5, 2)), num_warmup=1, num_samples=1, progress_bar=False, print_summary=False)
    with pytest.raises(ValueError):
        m.fit(0, np.ones(5), np.ones((5, 3)), num_warmup=1, num_samples=1, progress_bar=False, print_summary=False)
    with pytest.raises(ValueError):
        m.fit(0, np.ones(5), np.ones((4, 2)), num_warmup=1, num_samples=1, progress_bar=False, print_summary=False)
    with pytest.raises(ValueError):
        m.predict(0, np.ones((5, 2)), m.from_flat(np.zeros((1, 14))) | {"noise": np.ones(1)})
    X, y = m._set_data(np.ones(5), np.arange(5.0))           # one y column is broadcast over the outputs
    assert y.shape == (5, 2) and np.array_equal(y[:, 1], np.arange(5.0))


def test_bindings_check_shapes_before_calling_the_library():
    """Context.bnn_loglik / bnn_predict compare params, y and eps with the network; nothing of the context is touched
    before the check, so a bare instance shows it"""
    from gpax_b200 import _ffi
    ctx = object.__new__(_ffi.Context)
    X, y, widths = np.ones((4, 2)), np.ones((4, 1)), [3, 1]
    good = np.zeros(2 * 3 + 3 + 3 + 1)
    with pytest.raises(ValueError):
        ctx.bnn_loglik(X, y, widths, 1, good[:-1], 0.1)                    # params for another network
    with pytest.raises(ValueError):
        ctx.bnn_loglik(np.ones((4, 1)), y, widths, 1, good, 0.1)           # X with one column: 10 parameters, not 13
    with pytest.raises(ValueError):
        ctx.bnn_loglik(X, np.ones((4, 2)), widths, 1, good, 0.1)           # y with the wrong output count
    with pytest.raises(ValueError):
        ctx.bnn_loglik(X, np.ones((3, 1)), widths, 1, good, 0.1)           # y with the wrong row count
    with pytest.raises(ValueError):
        ctx.bnn_predict(X, widths, 1, np.zeros((2, good.size + 1)))
    with pytest.raises(ValueError):
        ctx.bnn_predict(X, widths, 1, np.zeros((2, good.size)), [0.1, 0.1], np.zeros((2, 1, 3, 1)))


def test_refusals():
    from gpax_b200 import BNN
    with pytest.raises(NotImplementedError):
        BNN(1, 1, nn=lambda X, p: X)
    with pytest.raises(NotImplementedError):
        BNN(1, 1, nn_prior=lambda: {})


class _Dev:
    def __init__(self, a):
        self.a = a

    def free(self):
        pass


class _StubCtx:
    """stands in for _ffi.Context: the oracle's likelihood and predictive forward pass, and a record of what predict got"""

    def to_device(self, a):
        return _Dev(np.asarray(a))

    def bnn_loglik(self, Xd, yd, widths, act, flat, sigma):
        v, gs, gp, _ = bo.loglik(Xd.a, yd.a, Xd.a.shape[1], list(widths), flat, sigma)
        return v, gs, gp

    def bnn_predict(self, X, widths, act, params, sigma=None, eps=None):
        self.eps = eps
        return bo.predict(np.asarray(X), np.asarray(X).shape[1], list(widths), params, sigma, eps)


@pytest.mark.parametrize("noise_prior", [None, "halfnormal"])
def test_log_joint_against_finite_differences(noise_prior):
    from gpax_b200 import BNN
    from gpax_b200 import priors as P
    from gpax_b200.bnn import BNNLogJoint
    pr = P.HalfNormal(0.5) if noise_prior else None
    m = BNN(2, 1, noise_prior_dist=pr, hidden_dim=[3], ctx=_StubCtx())
    rng = np.random.default_rng(3)
    X, y = rng.uniform(-1, 1, (7, 2)), rng.standard_normal((7, 1))
    lj = BNNLogJoint(m, X, y, rng)
    u = lj.init_u()
    assert u.shape == (lj.dim,) == (1 + 2 * 3 + 3 + 3 + 1,)
    u = u + 0.1 * rng.standard_normal(u.size)
    for jac in (False, True):
        v, g = lj(u, jac)
        h = 1e-6
        num = np.array([(lj(u + h * e, jac)[0] - lj(u - h * e, jac)[0]) / (2 * h) for e in np.eye(u.size)])
        np.testing.assert_allclose(g, num, rtol=1e-6, atol=1e-7 * np.abs(num).max())
    # the terms themselves: likelihood + noise prior (+ log|dsigma/du|) + Normal weights + Cauchy biases
    noise = pr or P.LogNormal(0.0, 1.0)
    sigma = float(noise.transform(u[0]))
    flat = u[1:]
    mask = m._weight_mask()
    want = (bo.loglik(X, y, 2, [3, 1], flat, sigma)[0] + float(noise.log_prob(sigma)) + float(noise.log_abs_jac(u[0]))
            + float(np.sum(P.Normal(0, 1).log_prob(flat[mask]))) + float(np.sum(P.Cauchy(0, 1).log_prob(flat[~mask]))))
    assert abs(lj(u, True)[0] - want) <= 1e-12 * abs(want)
    d = lj.to_dict(np.stack([u, u]))
    assert d["w0"].shape == (2, 2, 3) and d["noise"].shape == (2,) and d["noise"][0] == sigma


def test_log_joint_rejects_non_finite():
    from gpax_b200 import BNN
    from gpax_b200.bnn import BNNLogJoint
    m = BNN(1, 1, hidden_dim=[2], ctx=_StubCtx())
    lj = BNNLogJoint(m, np.zeros((3, 1)), np.zeros((3, 1)), np.random.default_rng(0))
    u = lj.init_u()
    u[0] = 1e6        # sigma overflows
    v, g = lj(u, True)
    assert v == -np.inf and np.all(g == 0)


def test_predict_eps_stream_is_the_reference_per_draw_stream():
    """draw s uses jax.random.split(key, S)[s] and jax.random.normal(that key, (n, P, O))"""
    from gpax_b200 import BNN, prng
    ctx = _StubCtx()
    m = BNN(1, 2, hidden_dim=[3], ctx=ctx)
    S, n, Pn = 3, 2, 5
    samples = m.from_flat(_flat(1, [3, 2], 4)[None] * np.array([[1.0], [0.9], [1.1]]))
    samples["noise"] = np.array([0.1, 0.2, 0.3])
    key = prng.PRNGKey(7)
    mean, ys = m.predict(key, np.linspace(-1, 1, Pn), samples, n=n)
    keys = prng.split(key, S)
    for s in range(S):
        np.testing.assert_array_equal(ctx.eps[s], prng.normal(keys[s], (n, Pn, 2)).astype(np.float64))
    assert mean.shape == (Pn, 2) and ys.shape == (S, Pn, 2)
    loc, y1 = m.sample_single_posterior_predictive(key, np.linspace(-1, 1, Pn), {k: v[0] for k, v in samples.items()}, n)
    np.testing.assert_array_equal(ctx.eps[0], prng.normal(key, (n, Pn, 2)).astype(np.float64))
    assert loc.shape == y1.shape == (Pn, 2)
