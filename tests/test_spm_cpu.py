"""sPM on the CPU (the model, its log joint and its NUTS fit are host code): SPMLogJoint's value and gradient against the
closed form and against central differences, recovery of a linear model's parameters, sample shapes, vectorized chains
against sequential ones, get_param_means, predict's random stream, the noise priors, and X reaching the model unreshaped.
The last tests run the reference's own test_spm.py model and program after `from gpax_b200 import priors as numpyro`."""
import math

import numpy as np
import pytest

from gpax_b200 import priors as numpyro
from gpax_b200 import priors as P
from gpax_b200.spm import SPMLogJoint, sPM
from gpax_b200.utils import get_keys, posterior_eps


def linear(x, params):
    return params["a"] * x + params["b"]


def linear_prior():
    a = numpyro.sample("a", numpyro.distributions.Normal(0, 5))
    b = numpyro.sample("b", numpyro.distributions.Normal(1, 4))
    return {"a": a, "b": b}


def linear_data(N=32, seed=0):
    rng = np.random.default_rng(seed)
    X = np.linspace(0, 1, N)
    return X, 2 * X + 3 + 0.1 * rng.standard_normal(N)


def _normal_lp(t, loc, scale):
    return -0.5 * ((t - loc) / scale) ** 2 - math.log(scale) - 0.5 * math.log(2 * math.pi)


def _closed_form(X, y, u, noise_prior):
    """value and gradient of the linear model's log joint (with the Jacobian of sigma = exp(u_2)) written out by hand"""
    a, b, sigma = u[0], u[1], math.exp(u[2])
    r = y - (a * X + b)
    val = float(np.sum(_normal_lp(y, a * X + b, sigma))) + _normal_lp(a, 0, 5) + _normal_lp(b, 1, 4)
    val += float(noise_prior.log_prob(sigma)) + u[2]
    g = np.array([np.sum(r * X) / sigma ** 2 - a / 25,
                  np.sum(r) / sigma ** 2 - (b - 1) / 16,
                  (np.sum(r * r / sigma ** 3 - 1 / sigma) + float(noise_prior.dlog_prob(sigma))) * sigma + 1.0])
    return val, g


@pytest.mark.parametrize("noise_dist", [None, P.HalfNormal(0.5), P.Gamma(2.0, 8.0)])
def test_log_joint_against_closed_form_and_central_differences(noise_dist):
    X, y = linear_data(20)
    lj = SPMLogJoint(sPM(linear, linear_prior, noise_prior_dist=noise_dist), X, y)
    assert [s.name for s in lj.sites] == ["a", "b", "noise"] and lj.dim == 3
    assert list(lj.model_coord) == [True, True, False]
    prior = noise_dist if noise_dist is not None else P.LogNormal(0, 1)
    for u in (np.array([1.5, 2.0, math.log(0.3)]), np.array([-0.7, 4.1, math.log(1.7)])):
        val, g = lj(u, jacobian=True)
        val_ref, g_ref = _closed_form(X, y, u, prior)
        assert abs(val - val_ref) <= 1e-12 * abs(val_ref)
        np.testing.assert_allclose(g, g_ref, rtol=1e-7, atol=1e-7 * np.abs(g_ref).max())
        h = 1e-5
        num = np.array([(lj(u + h * e, True)[0] - lj(u - h * e, True)[0]) / (2 * h) for e in np.eye(3)])
        np.testing.assert_allclose(g, num, rtol=1e-6, atol=1e-6 * np.abs(num).max())
        # without the Jacobian: the value drops log sigma, the noise coordinate's gradient drops 1
        v0, g0 = lj(u, jacobian=False)
        assert abs(v0 - (val - u[2])) <= 1e-12 * abs(val)
        np.testing.assert_allclose(g0, g - np.array([0, 0, 1.0]), rtol=1e-12, atol=1e-12)


def test_log_joint_refuses_non_positive_noise():
    X, y = linear_data(8)
    lj = SPMLogJoint(sPM(linear, linear_prior, noise_prior_dist=P.Normal(0, 1)), X, y)
    val, g = lj(np.array([1.0, 1.0, -0.2]), jacobian=True)
    assert val == -np.inf and np.array_equal(g, np.zeros(3))


def test_init_to_median():
    X, y = linear_data(8)
    lj = SPMLogJoint(sPM(linear, linear_prior, noise_prior_dist=P.LogNormal(0.5, 2.0)), X, y)
    np.testing.assert_allclose(lj.init_u(), [0.0, 1.0, 0.5], atol=1e-15)


@pytest.fixture(scope="module")
def linear_fit():
    X, y = linear_data()
    m = sPM(linear, linear_prior)
    m.fit(get_keys(3)[0], X, y, num_warmup=300, num_samples=300, num_chains=2, progress_bar=False, print_summary=False)
    return m, X, y


def test_nuts_recovers_the_linear_model(linear_fit):
    m, X, y = linear_fit
    s = m.get_samples()
    for k, true in (("a", 2.0), ("b", 3.0)):
        assert abs(s[k].mean() - true) < 4 * s[k].std(), (k, s[k].mean(), s[k].std())
        assert s[k].std() < 0.2
    assert 0.05 < s["noise"].mean() < 0.2


def test_sample_shapes_and_mu(linear_fit):
    m, X, _ = linear_fit
    s = m.get_samples()
    assert set(s) == {"a", "b", "noise", "mu"}
    assert s["a"].shape == s["b"].shape == s["noise"].shape == (600,)
    assert s["mu"].shape == (600, X.shape[0])
    c = m.get_samples(chain_dim=True)
    assert c["a"].shape == (2, 300) and c["mu"].shape == (2, 300, X.shape[0])
    # mu is the model at each kept draw
    np.testing.assert_allclose(c["mu"][1, 7], c["a"][1, 7] * X + c["b"][1, 7], rtol=1e-15)
    np.testing.assert_array_equal(s["mu"], c["mu"].reshape(600, -1))


def test_mu_is_written_once_per_kept_draw():
    X, y = linear_data(8)
    calls = []

    def counted(x, params):
        calls.append(1)
        return linear(x, params)
    m = sPM(counted, linear_prior)
    m.fit(1, X, y, num_warmup=20, num_samples=15, num_chains=2, progress_bar=False, print_summary=False)
    evals = m.mcmc.stats[-1]["grad_evals"]
    # one model call per evaluation plus two per model coordinate (central differences), then one per kept draw
    assert len(calls) == evals * (1 + 2 * 2) + 2 * 15


def test_get_param_means_skips_mu(linear_fit):
    m, _, _ = linear_fit
    means = m.get_param_means()
    assert set(means) == {"a", "b", "noise"}
    assert all(type(v) is float for v in means.values())
    assert means["a"] == m.get_samples()["a"].mean()


def test_vectorized_chains_equal_sequential():
    X, y = linear_data(16)
    out = []
    for method in ("sequential", "vectorized"):
        m = sPM(linear, linear_prior)
        m.fit(get_keys(1)[0], X, y, num_warmup=40, num_samples=30, num_chains=3, chain_method=method,
              progress_bar=False, print_summary=False)
        out.append(m.get_samples(chain_dim=True))
    assert set(out[0]) == set(out[1])
    for k in out[0]:
        assert np.array_equal(out[0][k], out[1][k]), k


def _fixed_samples(S=6):
    rng = np.random.default_rng(5)
    return {"a": rng.normal(2, 0.1, S), "b": rng.normal(3, 0.1, S), "noise": rng.uniform(0.05, 0.3, S)}


@pytest.mark.parametrize("n", [1, 4])
def test_predict_is_loc_plus_noise_times_mean_eps(n):
    s = _fixed_samples()
    Xn = np.linspace(-1, 2, 7)
    key = get_keys(2)[1]
    m = sPM(linear, linear_prior)
    y_pred, y_sampled = m.predict(key, Xn, s, n=n)
    loc = s["a"][:, None] * Xn + s["b"][:, None]
    eps = posterior_eps(key, 6, n, 7)
    assert y_pred.shape == (7,) and y_sampled.shape == (6, 7)
    np.testing.assert_allclose(y_pred, loc.mean(0), rtol=1e-15)
    np.testing.assert_allclose(y_sampled, loc + s["noise"][:, None] * eps.mean(1), rtol=1e-14)
    # take_point_predictions_mean=False keeps every draw's loc
    loc_all, y2 = m.predict(key, Xn, s, n=n, take_point_predictions_mean=False)
    np.testing.assert_allclose(loc_all, loc, rtol=1e-15)
    np.testing.assert_array_equal(y2, y_sampled)


def test_predict_filter_nans():
    s = _fixed_samples()
    s["a"][2] = np.nan
    Xn = np.linspace(0, 1, 5)
    m = sPM(linear, linear_prior)
    _, y_all = m.predict(0, Xn, s)
    assert y_all.shape == (6, 5) and np.isnan(y_all[2]).all()
    _, y = m.predict(0, Xn, s, filter_nans=True)
    assert y.shape == (5, 5) and not np.isnan(y).any()
    np.testing.assert_array_equal(y, y_all[[0, 1, 3, 4, 5]])


def test_sample_single_posterior_predictive():
    s = {k: v[0] for k, v in _fixed_samples().items()}
    Xn = np.linspace(0, 1, 5)
    key = get_keys(4)[0]
    loc, y = sPM(linear, linear_prior).sample_single_posterior_predictive(key, Xn, s, 3)
    eps = posterior_eps(key, 1, 3, 5, per_draw_keys=False)[0]
    np.testing.assert_allclose(loc, s["a"] * Xn + s["b"], rtol=1e-15)
    np.testing.assert_allclose(y, loc + s["noise"] * eps.mean(0), rtol=1e-14)


def test_noise_prior_dist_is_the_noise_site():
    X, y = linear_data(8)
    hn = P.HalfNormal(0.25)
    lj = SPMLogJoint(sPM(linear, linear_prior, noise_prior_dist=hn), X, y)
    assert lj.sites[-1].name == "noise" and lj.sites[-1].prior is hn
    draws = sPM(linear, linear_prior, noise_prior_dist=hn)
    draws.fit(0, X, y, num_warmup=30, num_samples=30, progress_bar=False, print_summary=False)
    assert np.all(draws.get_samples()["noise"] > 0)


def test_noise_prior_program_warns_and_is_honoured():
    X, y = linear_data(12)

    def noise_prior():
        return numpyro.sample("noise", numpyro.distributions.HalfNormal(0.3))
    with pytest.warns(FutureWarning, match="noise_prior"):
        m = sPM(linear, linear_prior, noise_prior=noise_prior)
    lj = SPMLogJoint(m, X, y)
    ref = SPMLogJoint(sPM(linear, linear_prior, noise_prior_dist=P.HalfNormal(0.3)), X, y)
    u = np.array([1.2, 2.5, math.log(0.2)])
    v, g = lj(u, True)
    v_ref, g_ref = ref(u, True)
    assert v == v_ref
    np.testing.assert_allclose(g, g_ref, rtol=1e-8)


def test_sample_from_prior():
    X = np.linspace(0, 1, 9)
    m = sPM(linear, linear_prior)
    y = m.sample_from_prior(get_keys(0)[0], X, num_samples=400)
    assert y.shape == (400, 9)
    np.testing.assert_array_equal(y, m.sample_from_prior(get_keys(0)[0], X, num_samples=400))
    # y(0) = b + noise * eps with b ~ Normal(1, 4): the prior-predictive mean is 1
    assert abs(y[:, 0].mean() - 1.0) < 4 * 4 / math.sqrt(400) + 0.5


@pytest.mark.parametrize("X", [np.linspace(0, 1, 10), np.linspace(0, 1, 10)[:, None]])
def test_x_reaches_the_model_unreshaped(X):
    seen = []

    def model(x, params):
        seen.append(np.shape(x))
        return params["a"] * np.asarray(x).sum(-1) if np.ndim(x) == 2 else params["a"] * x + params["b"]
    y = 2 * np.asarray(X).reshape(10) + 3
    m = sPM(model, linear_prior)
    m.fit(0, X, y, num_warmup=5, num_samples=5, progress_bar=False, print_summary=False)
    assert set(seen) == {X.shape}
    seen.clear()
    Xn = X[:4]
    m.predict(0, Xn)
    assert set(seen) == {Xn.shape}


# ---- the reference's tests/test_spm.py model and program, unchanged but for the import above
def get_dummy_data():
    X = np.linspace(1, 2, 8) + 0.1 * np.random.default_rng(0).standard_normal(8)
    return X, 10 * X ** 2


def model(x, params):
    return params["a"] * x ** params["b"]


def model_priors():
    a = numpyro.sample("a", numpyro.distributions.LogNormal(0, 1))
    b = numpyro.sample("b", numpyro.distributions.Normal(3, 1))
    return {"a": a, "b": b}


def test_reference_program_fit_get_samples_predict():
    key1, key2 = get_keys()
    X, y = get_dummy_data()
    X_test = np.linspace(X.min(), X.max(), 200)
    m = sPM(model, model_priors)
    m.fit(key1, X, y, num_warmup=100, num_samples=100, progress_bar=False, print_summary=False)
    assert m.mcmc is not None
    samples = m.get_samples()
    for k, v in samples.items():
        assert isinstance(k, str) and isinstance(v, np.ndarray) and len(v) == 100
    y_mean, y_sampled = m.predict(key2, X_test)
    assert y_mean.shape == X_test.shape and y_sampled.shape == (100, 200)


def test_reference_prediction_with_given_samples():
    rng = np.random.default_rng(1)
    samples = {"a": rng.standard_normal(100), "b": rng.standard_normal(100), "noise": rng.standard_normal(100)}
    X_test = np.linspace(1, 2, 200)
    y_mean, y_sampled = sPM(model, model_priors).predict(get_keys()[1], X_test, samples)
    assert y_mean.shape == (200,) and y_sampled.shape == (100, 200)
