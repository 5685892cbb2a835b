"""User kernel and mean functions without a GPU: the function setters of gpax/utils/fn.py (the reference's
test_func_setter.py cases, on NumPy), GramLogJoint over a NumPy stand-in for b2gp_mll_gram, and the draw chunking of
the callable-kernel posterior."""
import numpy as np
import pytest

import oracle
from gpax_b200 import priors as P
from gpax_b200.gp import ExactGP, gram_chunks
from gpax_b200.inference import GramLogJoint, make_log_joint
from gpax_b200.kernels import RBFKernel
from gpax_b200.utils import _set_noise_kernel_fn, set_fn, set_kernel_fn
from gpax_b200.vigp import viGP


# ------------------------------------------------------------------ function setters
def linear_kernel_test(X, Z, k_scale):
    return k_scale * np.dot(X, Z.T)


def rbf_test(X, Z, k_length, k_scale):
    scaled_X = X / k_length
    scaled_Z = Z / k_length
    X2 = (scaled_X ** 2).sum(1, keepdims=True)
    Z2 = (scaled_Z ** 2).sum(1, keepdims=True)
    r2 = X2 - 2 * scaled_X @ scaled_Z.T + Z2.T
    return k_scale * np.exp(-0.5 * r2)


def sample_function(x, a, b):
    return a + b * x


def test_set_fn():
    assert set_fn(sample_function)(2, {"a": 1, "b": 3}) == 7


def test_set_kernel_fn():
    lin, rbf = set_kernel_fn(linear_kernel_test), set_kernel_fn(rbf_test, jit_decorator=False)
    X = np.array([[1.0, 2], [3, 4], [5, 6]])
    Z = np.array([[1.0, 2], [3, 4]])
    assert np.array_equal(linear_kernel_test(X, Z, 1.0), lin(X, Z, {"k_scale": 1.0}))
    assert np.array_equal(rbf_test(X, Z, 1.0, 1.0), rbf(X, Z, {"k_length": 1.0, "k_scale": 1.0}))


def test_set_kernel_fn_with_jitter():
    jitter = 1e-5
    lin, rbf = set_kernel_fn(linear_kernel_test), set_kernel_fn(rbf_test)
    X = np.array([[1.0, 2], [3, 4], [5, 6]])
    assert np.array_equal(linear_kernel_test(X, X, 1.0) + jitter * np.eye(3), lin(X, X, {"k_scale": 1.0}, jitter=jitter))
    assert np.array_equal(rbf_test(X, X, 1.0, 1.0) + jitter * np.eye(3), rbf(X, X, {"k_length": 1.0, "k_scale": 1.0}, jitter=jitter))
    assert np.array_equal(lin(X, X, {"k_scale": 1.0}, noise=0.5, jitter=0.0), linear_kernel_test(X, X, 1.0) + 0.5 * np.eye(3))


def test_set_noise_kernel_fn():
    """on a user function (source-free key mapping); this package's fused RBFKernel is covered on the GPU"""
    seen = {}

    def k(X, Z, params, noise=0, jitter=1e-6):
        seen.update(params)
        return oracle.rbf_kernel(X, Z, params, noise, jitter)
    X = np.array([[1.0, 2], [3, 4], [5, 6]])
    params = {"k_noise_length": np.array([1.0]), "k_noise_scale": np.array(1.0), "k_length": 7.0, "other": 3}
    got = _set_noise_kernel_fn(k)(X, X, params)
    assert np.array_equal(got, oracle.rbf_kernel(X, X, {"k_length": np.array([1.0]), "k_scale": np.array(1.0)}))
    assert seen == {"k_length": params["k_noise_length"], "k_scale": params["k_noise_scale"], "other": 3}
    assert _set_noise_kernel_fn(RBFKernel).__name__ == "RBFKernel"


# ------------------------------------------------------------------ GramLogJoint over a NumPy b2gp_mll_gram
class FakeCtx:
    """b2gp_mll_gram restated on NumPy; keeps the derivative matrices of the last call"""

    def mll_gram(self, K, y, dKs=(), want_grad=True, want_alpha=False):
        self.dKs = [np.array(D) for D in dKs]
        Ks = 0.5 * (K + K.T)
        L = np.linalg.cholesky(Ks)
        alpha = np.linalg.solve(Ks, y)
        val = -0.5 * y @ alpha - np.log(np.diag(L)).sum() - 0.5 * len(y) * np.log(2 * np.pi)
        W = np.outer(alpha, alpha) - np.linalg.inv(Ks)
        grad = np.array([0.5 * np.sum(W * D) for D in dKs]) if want_grad else None
        return val, grad, (alpha if want_alpha else None), 0


class Counting:
    def __init__(self, fn=oracle.rbf_kernel):
        self.fn, self.calls, self.params = fn, 0, []

    def __call__(self, X, Z, params, noise=0, jitter=1e-6, **kw):
        self.calls += 1
        self.params.append(dict(params))
        return self.fn(X, Z, params, noise, jitter)


def _model(kernel, input_dim=2, cls=ExactGP, N=30, cols=2, **kw):
    rng = np.random.default_rng(0)
    m = cls(input_dim, kernel, ctx=FakeCtx(), **kw)
    m.X_train = rng.uniform(0, 1, (N, cols))
    m.y_train = np.sin(3 * m.X_train[:, 0]) + 0.1 * rng.standard_normal(N)
    return m


@pytest.mark.parametrize("cls", [ExactGP, viGP])
def test_sites_and_dispatch(cls):
    k = Counting()
    m = _model(k, cls=cls)
    lj = make_log_joint(m)
    assert isinstance(lj, GramLogJoint)
    assert [(s.name, s.shape) for s in lj.sites] == [("k_length", (2,)), ("k_scale", ()), ("noise", ())]
    lj(lj.init_u(), True)
    assert all(p["period"] is None for p in k.params)
    assert set(k.params[0]) == {"k_length", "k_scale", "period"}


def test_kernel_dim_sets_the_ard_plate():
    k = Counting(lambda X, Z, p, noise, jitter: oracle.rbf_kernel(X[:, :1], Z[:, :1], p, noise, jitter))
    lj = make_log_joint(_model(k, input_dim=1, cols=2))
    assert dict((s.name, s.shape) for s in lj.sites)["k_length"] == (1,)
    lj(lj.init_u(), True)
    assert np.asarray(k.params[0]["k_length"]).shape == (1,)


def test_fd_derivatives_match_analytic_rbf():
    m = _model(Counting())
    lj = make_log_joint(m)
    u = lj.init_u() + np.array([0.2, -0.3, 0.1, -0.4])
    lj(u, True)
    th = np.exp(u)                                    # LogNormal sites: u = log theta
    X = m.X_train
    K0 = oracle.rbf_kernel(X, X, {"k_length": th[:2], "k_scale": th[2]}, 0.0, 0.0)
    ana = [K0 * (X[:, k][:, None] - X[:, k][None, :]) ** 2 / th[k] ** 2 for k in range(2)] + [K0, th[3] * np.eye(len(X))]
    assert len(m.ctx.dKs) == 4
    for got, ref in zip(m.ctx.dKs, ana):
        np.testing.assert_allclose(got, ref, rtol=1e-7, atol=1e-7 * np.abs(ref).max())


def test_mean_coordinates_take_no_kernel_evaluations():
    def mean_fn(X, p):
        return p["m0"] + p["m1"] * X[:, 0]

    def mprior():
        return {"m0": P.sample("m0", P.Normal(0.0, 1.0)), "m1": P.sample("m1", P.Normal(0.0, 1.0))}
    k = Counting()
    m = _model(k, input_dim=1, cols=1, mean_fn=mean_fn, mean_fn_prior=mprior)
    lj = make_log_joint(m)
    assert [s.name for s in lj.sites] == ["k_length", "k_scale", "noise", "m0", "m1"]
    k.calls = 0
    val, g = lj(lj.init_u(), True)
    assert k.calls == 1 + 2 * 3 and len(m.ctx.dKs) == 3
    # the mean coordinates' gradient is alpha . dm/du, checked by central differences of the whole log joint
    u, h = lj.init_u(), 1e-5
    for c in (3, 4):
        e = np.zeros(lj.dim)
        e[c] = h
        fd = (lj(u + e, True)[0] - lj(u - e, True)[0]) / (2 * h)
        np.testing.assert_allclose(g[c], fd, rtol=1e-6)


# ------------------------------------------------------------------ draw chunking
def test_gram_chunks_budget():
    N, P = 100, 20
    per = 8 * (N * N + P * N + P * P)
    assert gram_chunks(10, N, P, True, budget=3 * per) == [(0, 3), (3, 6), (6, 9), (9, 10)]
    assert gram_chunks(10, N, P, True, budget=per - 1) == [(s, s + 1) for s in range(10)]
    assert gram_chunks(7, N, P, False, budget=8 * (N * N + P * N + P) * 7) == [(0, 7)]
    for S in (1, 5, 33):
        ch = gram_chunks(S, 300, 50, True, budget=10 * 8 * (300 * 300 + 50 * 300 + 2500))
        assert ch[0][0] == 0 and ch[-1][1] == S and all(b - a <= 10 for a, b in ch)
        assert all(ch[i][1] == ch[i + 1][0] for i in range(len(ch) - 1))
