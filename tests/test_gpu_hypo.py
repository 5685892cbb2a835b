"""Hypothesis learning with the GP-wrapped model on the GPU: hypo.step(gp_wrap=True) fits an ExactGP whose mean function is
the candidate model (its likelihood evaluations on b2gp_mll), its objective against ExactGP.predict called directly with
the same key, and a two-model hypothesis-learning loop (step per model, update_record, sample_next) end to end."""
import numpy as np
import pytest

import gpax_b200
from gpax_b200 import priors as numpyro
from gpax_b200.hypo import sample_next, step, update_record
from gpax_b200.utils import get_keys

pytestmark = pytest.mark.gpu


def power_law(x, params):
    return params["a"] * x ** params["b"]


def power_law_priors():
    a = numpyro.sample("a", numpyro.distributions.LogNormal(0, 1))
    b = numpyro.sample("b", numpyro.distributions.Normal(3, 1))
    return {"a": a, "b": b}


def line(x, params):
    return params["c"] * x + params["d"]


def line_priors():
    c = numpyro.sample("c", numpyro.distributions.Normal(0, 10))
    d = numpyro.sample("d", numpyro.distributions.Normal(0, 10))
    return {"c": c, "d": d}


def get_dummy_data():
    X = np.linspace(1, 2, 8) + 0.1 * np.random.default_rng(0).standard_normal(8)
    return X, 10 * X ** 2


def test_step_gp_wrap_fits_an_exact_gp_on_the_gpu(monkeypatch):
    ctx = gpax_b200.default_context()
    calls = []
    mll = ctx.mll

    def counted(*a, **kw):
        calls.append(1)
        return mll(*a, **kw)
    monkeypatch.setattr(ctx, "mll", counted)
    X, y = get_dummy_data()
    Xu = np.linspace(1, 3, 12)
    obj, m = step(power_law, power_law_priors, X, y, Xu, gp_wrap=True, num_warmup=60, num_samples=60, print_summary=False)
    assert isinstance(m, gpax_b200.ExactGP) and m.mean_fn is power_law and m.mean_fn_prior is power_law_priors
    assert len(calls) > 0
    s = m.get_samples()
    assert {"a", "b", "k_length", "k_scale", "noise"} <= set(s)
    assert s["a"].shape == (60,) and s["k_length"].shape == (60, 1)
    # obj is the variance over draws of ExactGP.predict with the key of the last fit
    assert isinstance(obj, np.ndarray) and obj.shape == (12,)
    _, y_sampled = m.predict(get_keys(0)[0], Xu)
    assert y_sampled.shape == (60, 1, 12)
    np.testing.assert_allclose(obj, y_sampled.squeeze().var(0), rtol=1e-12, atol=0)


def test_reference_step_gp_wrap():
    X, y = get_dummy_data()
    obj, _ = step(power_law, power_law_priors, X, y, X, gp_wrap=True, num_warmup=50, num_samples=50)
    assert isinstance(obj, np.ndarray) and obj.shape == X.shape


def test_two_model_hypothesis_learning_loop():
    """arXiv:2112.06649's loop: pick a model by softmax over the running rewards, fit it (GP-wrapped) on the measured
    points, reward it when its predictive uncertainty over the unmeasured points fell, measure where it is largest"""
    rng = np.random.default_rng(1)
    X_all = np.linspace(1, 2, 40)
    y_all = 10 * X_all ** 2 + 0.05 * rng.standard_normal(40)
    measured = list(rng.choice(40, 6, replace=False))
    models = [(power_law, power_law_priors), (line, line_priors)]
    record = np.zeros((2, 2))
    last_unc = [np.inf, np.inf]
    np.random.seed(0)
    chosen = []
    for _ in range(4):
        idx = int(sample_next(record[:, 1], "softmax", temperature=0.3))
        chosen.append(idx)
        unmeasured = np.setdiff1d(np.arange(40), measured)
        obj, m = step(*models[idx], X_all[measured], y_all[measured], X_all[unmeasured], gp_wrap=True,
                      num_warmup=40, num_samples=40, print_summary=False)
        assert obj.shape == (unmeasured.size,) and np.all(np.isfinite(obj))
        unc = float(obj.mean())
        update_record(record, idx, 1 if unc < last_unc[idx] else 0)
        last_unc[idx] = unc
        measured.append(int(unmeasured[int(obj.argmax())]))
    assert record[:, 0].sum() == 4 and len(set(measured)) == 10
    assert np.all((record[:, 1] >= 0) & (record[:, 1] <= 1))
