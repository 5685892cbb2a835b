"""CPU: the derivatives behind optimize_acq, pinned by central differences (no JAX here to pin them to).

- oracle.grad_oracle's d mean / dx and d var / dx against central differences of oracle.exact_posterior_chol;
- the package's acquisition chain rule (gpax_b200.acquisition.acq_value_grad) and the oracle's against central
  differences of acq_oracle's acquisitions of the oracle posterior, for the moment form and the MCMC sample-moment form
  with injected eps;
- prng.randint and optimize.py's ensure_array."""
import numpy as np
import pytest

import oracle
from oracle import acq_oracle as ao
from oracle import grad_oracle as gro
from gpax_b200 import acquisition as acq
from gpax_b200 import prng

H = 1e-5


def problem(kernel, d, seed=0, N=40, P=5):
    rng = np.random.default_rng(seed + 10 * d)
    X = rng.uniform(-1, 1, (N, d))
    y = np.sin(2 * X).sum(1) + 0.05 * rng.standard_normal(N)
    Xn = rng.uniform(-1, 1, (P, d))
    params = {"k_length": np.linspace(0.5, 0.9, d), "k_scale": 1.3, "noise": 0.05, "period": 1.7}
    return X, y, Xn, params


def central(f, x, h=H):
    """central differences of f (scalar or array valued) w.r.t. the vector x: result [..., d]"""
    cols = []
    for k in range(x.size):
        e = np.zeros_like(x)
        e[k] = h
        cols.append((np.asarray(f(x + e)) - np.asarray(f(x - e))) / (2 * h))
    return np.stack(cols, -1)


@pytest.mark.parametrize("noiseless", [False, True])
@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("kernel", ["RBF", "Matern", "Periodic"])
def test_oracle_posterior_gradient_matches_central_differences(kernel, d, noiseless):
    X, y, Xn, params = problem(kernel, d)
    mean, var, dmean, dvar = gro.posterior_grad(X, y, Xn, params, kernel, noiseless)
    rm, rv = oracle.exact_posterior_chol(X, y, Xn, params, kernel, noiseless, diag_only=True)
    np.testing.assert_allclose(mean, rm, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(var, rv, rtol=1e-12, atol=1e-14)
    for p in range(Xn.shape[0]):
        def moments(x):
            Xq = Xn.copy()
            Xq[p] = x
            m, v = oracle.exact_posterior_chol(X, y, Xq, params, kernel, noiseless, diag_only=True)
            return np.array([m[p], v[p]])
        fd = central(moments, Xn[p].copy())
        scale = np.abs(fd).max()
        np.testing.assert_allclose(dmean[p], fd[0], rtol=1e-6, atol=1e-6 * scale, err_msg=f"dmean p={p}")
        np.testing.assert_allclose(dvar[p], fd[1], rtol=1e-6, atol=1e-6 * scale, err_msg=f"dvar p={p}")


def test_kernel_dx_is_the_derivative_of_the_gram_builders():
    for kernel in ("RBF", "Matern", "Periodic"):
        X, _, Xn, params = problem(kernel, 3, seed=5)
        D = gro.kernel_dx(Xn, X, params, kernel)
        kern = oracle.get_kernel(kernel)
        fd = central(lambda x: kern(x[None], X, params, jitter=0.0)[0], Xn[0].copy())   # [N, d]
        np.testing.assert_allclose(D[0].T, fd, rtol=1e-7, atol=1e-9, err_msg=kernel)


def acq_of_moments(kind, M, V, best_f, param, maximize):
    """acq_oracle's function of one point's moments; best_f None is the point's own mean (base_acq.py:59-60)"""
    m, v = np.array([M]), np.array([V])
    if kind == "EI":
        return ao.ei(m, v, best_f, maximize)[0]
    if kind == "POI":
        return ao.poi(m, v, best_f, param, maximize)[0]
    if kind == "UCB":
        return ao.ucb(m, v, param, maximize)[0]
    return ao.ue(m, v)[0]


CASES = [("EI", None, 0.0), ("EI", 0.3, 0.0), ("POI", None, 0.01), ("POI", -0.2, 0.05), ("UCB", None, 0.25),
         ("UCB", None, 4.0), ("UE", None, 0.0)]


@pytest.mark.parametrize("mcmc", [False, True])
@pytest.mark.parametrize("maximize", [False, True])
@pytest.mark.parametrize("kind,best_f,param", CASES)
def test_acquisition_chain_rule_matches_central_differences(kind, best_f, param, maximize, mcmc):
    X, y, Xn, params = problem("Matern", 2, seed=3)
    x0 = Xn[0].copy()
    draws = [params, dict(params, k_length=np.array([0.4, 0.7]), noise=0.08), dict(params, k_scale=0.9)] if mcmc else [params]
    eps = np.random.default_rng(7).standard_normal((len(draws), 4)) if mcmc else None

    def value(x):
        ms, vs = zip(*[oracle.exact_posterior_chol(X, y, x[None], p, "Matern", diag_only=True) for p in draws])
        if mcmc:
            ys = np.array(ms)[:, 0, None] + np.sqrt(np.array(vs)[:, 0, None]) * eps     # y = mean + chol(cov) eps, P = 1
            M, V = ao.moments_from_samples(ys.reshape(-1, 1))
            M, V = M[0], V[0]
        else:
            M, V = ms[0][0], vs[0][0]
        return acq_of_moments(kind, M, V, best_f, param, maximize)

    per = [gro.posterior_grad(X, y, x0[None], p, "Matern") for p in draws]
    m, v, dm, dv = (np.array([q[i][0] for q in per]) for i in range(4))
    got_v, got_g = acq.acq_value_grad(kind, m, v, dm, dv, eps, best_f, param, maximize)
    ref_v, ref_g = gro.acq_value_grad(kind, m, v, dm, dv, eps, best_f, param, maximize)
    fd = central(value, x0)
    assert np.isclose(got_v, value(x0), rtol=1e-12, atol=1e-15)
    scale = max(np.abs(fd).max(), 1e-12)
    np.testing.assert_allclose(got_g, fd, rtol=1e-6, atol=1e-6 * scale, err_msg="package chain rule")
    np.testing.assert_allclose(ref_g, fd, rtol=1e-6, atol=1e-6 * scale, err_msg="oracle chain rule")
    np.testing.assert_allclose(got_g, ref_g, rtol=1e-10, atol=1e-12 * scale)
    assert np.isclose(ref_v, got_v, rtol=1e-13)


def test_ei_with_best_f_none_at_one_point_is_sigma_phi0():
    """the reference's optimize_acq of EI with best_f=None: best_f is the point's own mean, u == 0"""
    val, g = acq.acq_value_grad("EI", [0.7], [0.09], [[1.0, -2.0]], [[0.3, 0.6]])
    assert np.isclose(val, 0.3 / np.sqrt(2 * np.pi), rtol=1e-15)
    np.testing.assert_allclose(g, np.array([0.3, 0.6]) / (2 * 0.3) / np.sqrt(2 * np.pi), rtol=1e-15)


def test_randint_is_deterministic_and_in_range():
    key = prng.PRNGKey(42)
    a = prng.randint(key, (1000,), 3, 17)
    assert a.dtype == np.int32 and a.shape == (1000,)
    assert np.array_equal(a, prng.randint(key, (1000,), 3, 17))
    assert a.min() >= 3 and a.max() < 17 and len(np.unique(a)) == 14
    assert not np.array_equal(a, prng.randint(prng.PRNGKey(43), (1000,), 3, 17))
    assert np.array_equal(prng.randint(key, (2, 3), 5, 5), np.full((2, 3), 5))        # span <= 0 -> minval
    assert np.array_equal(prng.randint(key, (4,), 5, 2), np.full(4, 5))
    one = prng.randint(key, (1,), 0, 100)
    assert one.shape == (1,) and 0 <= one[0] < 100


@pytest.mark.parametrize("span", [1000003, 1000])
def test_randint_restates_the_jax_04_reduction(span):
    """((hi % span) * ((2^16 % span)^2 % span) + lo % span) % span in uint32, words from the two halves of split(key)"""
    key = prng.PRNGKey(7)
    k1, k2 = prng.split(key, 2)
    hi = prng.random_bits(k1, 32, (64,)).astype(np.uint64)
    lo = prng.random_bits(k2, 32, (64,)).astype(np.uint64)
    mult = (((2 ** 16 % span) ** 2) % 2 ** 32) % span     # the square wraps in uint32: 0 for span > 2^16, as in JAX
    ref = ((((hi % span) * mult) % 2 ** 32 + lo % span) % 2 ** 32) % span
    np.testing.assert_array_equal(prng.randint(key, (64,), -5, span - 5), ref.astype(np.int64) - 5)


def test_ensure_array_follows_optimize_py():
    np.testing.assert_array_equal(acq.ensure_array(2.0), np.array([2.0]))
    np.testing.assert_array_equal(acq.ensure_array([1.0, 2.0]), np.array([1.0, 2.0]))
    np.testing.assert_array_equal(acq.ensure_array((1.0, -1.0)), np.array([1.0, -1.0]))
    a = np.array([0.5, 1.5])
    assert acq.ensure_array(a) is a
    for bad in (2, "2.0", None, {1: 2}):
        with pytest.raises(TypeError):
            acq.ensure_array(bad)


def test_new_functions_are_exported():
    for name in ("Thompson", "qKG", "optimize_acq"):
        assert name in acq.__all__ and callable(getattr(acq, name))


def test_optimize_acq_differentiates_only_the_plain_exact_posterior():
    """models whose predict() is not the exact-GP posterior inherit _posterior_grad but must take finite differences"""
    from gpax_b200 import ExactGP, MeasuredNoiseGP, UIGP, VarNoiseGP, vExactGP, viGP, viSparseGP
    for model in (ExactGP(2, "RBF"), viGP(2, "Matern")):
        assert acq._analytic_kind(acq.EI, model, {}) == "EI"
        assert acq._analytic_kind(acq.EI, model, {"penalty": "delta"}) is None
        assert acq._analytic_kind(acq.KG, model, {}) is None
    for model in (viSparseGP(2, "RBF"), MeasuredNoiseGP(2, "RBF"), VarNoiseGP(2, "RBF"), vExactGP(2, "RBF"), UIGP(2, "RBF")):
        assert acq._analytic_kind(acq.EI, model, {}) is None, type(model).__name__

    class MyGP(ExactGP):
        pass
    assert acq._analytic_kind(acq.UCB, MyGP(2, "RBF"), {}) is None
    assert acq._analytic_kind(acq.UCB, ExactGP(2, "RBF", mean_fn=lambda x: 0 * x[:, 0]), {}) is None
