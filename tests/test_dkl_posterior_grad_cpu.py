"""CPU: the derivative behind optimize_acq on viDKL / DKL, pinned by central differences (no JAX here to pin it to).

- dkl_grad_oracle.posterior_grad's d mean / dx and d var / dx w.r.t. the RAW test input against central differences of
  oracle.dkl_oracle.posterior, for ReLU and tanh networks with 1 and 3 hidden layers, the three kernels, D in {1, 6} and
  noiseless both ways.  Test points are kept away from ReLU's kink, where the central difference straddles it;
- which models and acquisitions acquisition.optimize_acq differentiates in closed form."""
import numpy as np
import pytest

from dkl_grad_oracle import posterior_grad
from gpax_b200 import acquisition as acq
from oracle import dkl_oracle as dko

H = 1e-5
MARGIN = 1e-3          # smallest |pre-activation| of a hidden unit at a test point (H moves it by ~1e-4 at most)


def problem(kind, act, D, hidden, seed=0, N=30, P=4):
    rng = np.random.default_rng(seed + 100 * D + 10 * len(hidden) + (act == "tanh"))
    widths = list(hidden) + [2]
    layers, i = [], D
    for w in widths:
        layers.append((rng.standard_normal((i, w)) / np.sqrt(i), 0.3 * rng.standard_normal(w)))
        i = w
    X = rng.uniform(-1, 1, (N, D))
    y = np.sin(2 * X).sum(1) + 0.05 * rng.standard_normal(N)
    rows = []
    while len(rows) < P:          # away from the kinks: every hidden pre-activation at least MARGIN from 0
        x = rng.uniform(-1, 1, (1, D))
        h, ok = x, True
        for W, b in layers[:-1]:
            pre = h @ W + b
            ok &= bool(np.abs(pre).min() > MARGIN)
            h = dko._act(pre, act)
        if ok or act == "tanh":
            rows.append(x[0])
    params = {"k_length": np.array([0.7, 1.1]), "k_scale": 1.3, "noise": 0.05, "period": 2.1}
    return X, y, np.array(rows), layers, params


def central(f, x, h=H):
    cols = []
    for k in range(x.size):
        e = np.zeros_like(x)
        e[k] = h
        cols.append((np.asarray(f(x + e)) - np.asarray(f(x - e))) / (2 * h))
    return np.stack(cols, -1)


@pytest.mark.parametrize("noiseless", [False, True])
@pytest.mark.parametrize("hidden", [(8,), (8, 7, 5)])
@pytest.mark.parametrize("D", [1, 6])
@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
def test_oracle_input_gradient_matches_central_differences(kind, act, D, hidden, noiseless):
    X, y, Xn, layers, params = problem(kind, act, D, hidden)
    mean, var, dmean, dvar = posterior_grad(kind, X, y, Xn, layers, act, params, noiseless)
    rm, rc = dko.posterior(kind, X, y, Xn, layers, act, params, noiseless)
    np.testing.assert_allclose(mean, rm, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(var, np.diag(rc), rtol=1e-8, atol=1e-12)
    assert dmean.shape == dvar.shape == (Xn.shape[0], D)
    for p in range(Xn.shape[0]):
        def moments(x):
            Xq = Xn.copy()
            Xq[p] = x
            m, c = dko.posterior(kind, X, y, Xq, layers, act, params, noiseless)
            return np.array([m[p], c[p, p]])
        fd = central(moments, Xn[p].copy())
        scale = np.abs(fd).max()
        np.testing.assert_allclose(dmean[p], fd[0], rtol=1e-6, atol=1e-6 * scale, err_msg=f"dmean p={p}")
        np.testing.assert_allclose(dvar[p], fd[1], rtol=1e-5, atol=1e-6 * scale, err_msg=f"dvar p={p}")


def test_relu_derivative_is_zero_at_zero():
    """jax.nn.relu's derivative at 0 is 0: a hidden unit that is exactly 0 passes no gradient"""
    W0 = np.array([[1.0, -1.0]])
    layers = [(W0, np.array([0.0, 0.5])), (np.array([[2.0], [3.0]]), np.zeros(1))]
    Hn = dko.mlp_forward(np.zeros((1, 1)), layers, "relu")
    from dkl_grad_oracle import input_vjp
    np.testing.assert_array_equal(input_vjp(Hn, layers, "relu", np.ones((1, 1))), [[-3.0]])


def test_optimize_acq_differentiates_dkl_models_with_one_channel():
    from gpax_b200 import DKL, viDKL, viMTDKL
    v, m = viDKL(6, 2), DKL(6, 2, hidden_dim=[8, 4])
    for model in (v, m):
        assert acq._analytic_kind(acq.EI, model, {}) == "EI", type(model).__name__
        assert acq._analytic_kind(acq.UCB, model, {}) == "UCB"
        assert acq._analytic_kind(acq.EI, model, {"penalty": "delta"}) is None
        assert acq._analytic_kind(acq.KG, model, {}) is None
        model.X_train, model.y_train = np.zeros((5, 6)), np.zeros(5)
        assert acq._analytic_kind(acq.POI, model, {}) == "POI"
    v.y_train = np.zeros((2, 5))                                    # two channels fitted side by side
    assert acq._analytic_kind(acq.EI, v, {}) is None
    assert acq._analytic_kind(acq.EI, viMTDKL(6, 2, num_latents=2), {}) is None

    class MyDKL(viDKL):
        pass
    assert acq._analytic_kind(acq.EI, MyDKL(6, 2), {}) is None
