"""Hypothesis learning on the CPU: the bandit policies and their refusals, update_record's running mean, split r-hat
against the formula written out here, and hypo.step on the standalone sPM -- the restart rule counted with a stand-in
`fit`, the objective's shape, and the reference's tests/test_hypo.py model and program after
`from gpax_b200 import priors as numpyro`."""
import numpy as np
import pytest
from scipy.stats import chi2

import gpax_b200
from gpax_b200 import priors as numpyro
from gpax_b200 import hypo
from gpax_b200.diagnostics import gelman_rubin, split_gelman_rubin
from gpax_b200.hypo import eps_greedy, sample_next, softmax, step, update_record
from gpax_b200.inference import MCMCResult
from gpax_b200.spm import sPM
from gpax_b200.utils import get_keys


def test_exports():
    assert gpax_b200.sPM is sPM and gpax_b200.sample_next is sample_next and gpax_b200.hypo is hypo
    assert "sPM" in gpax_b200.__all__ and "sample_next" in gpax_b200.__all__


# ---- bandit policies
def test_eps_greedy_with_eps_0_is_argmax():
    np.random.seed(0)
    r = np.array([0.3, 0.9, 0.1, 0.5])
    assert all(eps_greedy(r, eps=0.0) == 1 for _ in range(500))
    assert all(sample_next(r, "eps-greedy", eps=0.0) == 1 for _ in range(100))


def _chi2_ok(counts, probs, q=0.999):
    n = counts.sum()
    stat = float(np.sum((counts - n * probs) ** 2 / (n * probs)))
    return stat < chi2.ppf(q, len(probs) - 1), stat


def test_eps_greedy_with_eps_1_is_uniform():
    np.random.seed(1)
    r = np.array([0.3, 0.9, 0.1, 0.5])
    counts = np.bincount([eps_greedy(r, eps=1.0) for _ in range(4000)], minlength=4)
    ok, stat = _chi2_ok(counts, np.full(4, 0.25))
    assert ok, (counts, stat)


@pytest.mark.parametrize("temperature", [1.0, 0.5])
def test_softmax_frequencies_match_the_probabilities(temperature):
    np.random.seed(2)
    logits = np.array([0.0, 0.5, 1.0, -0.5])
    p = np.exp(logits / temperature) / np.exp(logits / temperature).sum()
    counts = np.bincount([softmax(logits, temperature) for _ in range(6000)], minlength=4)
    ok, stat = _chi2_ok(counts, p)
    assert ok, (counts, stat)
    np.random.seed(2)
    via_sample_next = [sample_next(logits, "softmax", temperature) for _ in range(50)]
    np.random.seed(2)
    assert via_sample_next == [softmax(logits, temperature) for _ in range(50)]


def test_policies_use_the_global_generator():
    r = np.array([0.0, 0.1, 0.2])
    np.random.seed(7)
    a = [sample_next(r, "softmax") for _ in range(20)] + [sample_next(r, "eps-greedy") for _ in range(20)]
    np.random.seed(7)
    b = [sample_next(r, "softmax") for _ in range(20)] + [sample_next(r, "eps-greedy") for _ in range(20)]
    assert a == b
    assert all(isinstance(i, (np.int64, int)) for i in a)


def test_sample_next_refusals():
    with pytest.raises(NotImplementedError):
        sample_next(np.array([0.0, 1.0]), "ucb")
    with pytest.raises(AttributeError):
        sample_next(np.zeros((2, 2)), "softmax")


def test_update_record_keeps_the_running_mean():
    record = np.zeros((3, 2))
    rewards = {0: [1.0, 0.0, 0.5, 2.0], 2: [3.0, -1.0]}
    for action, rs in rewards.items():
        for r in rs:
            out = update_record(record, action, r)
            assert out is record
    np.testing.assert_allclose(record[0], [4, np.mean(rewards[0])], rtol=1e-15)
    np.testing.assert_allclose(record[2], [2, np.mean(rewards[2])], rtol=1e-15)
    assert np.array_equal(record[1], [0, 0])


# ---- r-hat
def _rhat_by_hand(x):
    """R-hat of x [C, n] written out: W = mean within-chain variance, B/n = variance of the chain means (ddof 1)"""
    C, n = x.shape
    means = [sum(x[c]) / n for c in range(C)]
    within = [sum((v - means[c]) ** 2 for v in x[c]) / (n - 1) for c in range(C)]
    W = sum(within) / C
    grand = sum(means) / C
    B_n = sum((m - grand) ** 2 for m in means) / (C - 1)
    return np.sqrt(((n - 1) / n * W + B_n) / W)


def test_split_gelman_rubin_against_the_formula():
    x = np.random.default_rng(3).standard_normal((3, 11))
    half = 11 // 2
    split = np.concatenate([x[:, :half], x[:, -half:]])
    assert abs(float(split_gelman_rubin(x)) - _rhat_by_hand(split)) <= 1e-14
    assert abs(float(gelman_rubin(x)) - _rhat_by_hand(x)) <= 1e-14
    # one chain: its two halves are the chains
    y = np.random.default_rng(4).standard_normal((1, 8))
    assert abs(float(split_gelman_rubin(y)) - _rhat_by_hand(np.stack([y[0, :4], y[0, 4:]]))) <= 1e-14
    # trailing site dimensions are kept
    v = np.random.default_rng(5).standard_normal((2, 10, 3))
    r = split_gelman_rubin(v)
    assert r.shape == (3,)
    for j in range(3):
        s = np.concatenate([v[:, :5, j], v[:, -5:, j]])
        assert abs(r[j] - _rhat_by_hand(s)) <= 1e-14


def test_split_gelman_rubin_flags_shifted_chains():
    x = np.random.default_rng(6).standard_normal((4, 200))
    assert split_gelman_rubin(x) < 1.05
    x[1] += 3.0
    assert split_gelman_rubin(x) > 1.5
    drift = np.random.default_rng(7).standard_normal((1, 200)) + np.linspace(0, 6, 200)
    assert split_gelman_rubin(drift) > 1.5


# ---- step on sPM
def model(x, params):
    return params["a"] * x ** params["b"]


def model_priors():
    a = numpyro.sample("a", numpyro.distributions.LogNormal(0, 1))
    b = numpyro.sample("b", numpyro.distributions.Normal(3, 1))
    return {"a": a, "b": b}


def get_dummy_data():
    X = np.linspace(1, 2, 8) + 0.1 * np.random.default_rng(0).standard_normal(8)
    return X, 10 * X ** 2


def test_step_standalone_returns_the_predictive_variance():
    X, y = get_dummy_data()
    Xu = np.linspace(1, 3, 6)
    obj, m = step(model, model_priors, X, y, Xu, gp_wrap=False, num_warmup=50, num_samples=50, print_summary=False)
    assert isinstance(m, sPM) and isinstance(obj, np.ndarray) and obj.shape == (6,)
    _, samples = m.predict(get_keys(0)[0], Xu)
    np.testing.assert_array_equal(obj, samples.squeeze().var(0))


def test_step_without_unmeasured_points_returns_0():
    X, y = get_dummy_data()
    obj, m = step(model, model_priors, X, y, num_warmup=20, num_samples=20, print_summary=False)
    assert obj == 0 and isinstance(m, sPM)


def _fake_fit(log, rhat_ok):
    """a stand-in for sPM.fit: records the key, leaves samples whose split r-hat is below 1.1 when rhat_ok(call) holds"""
    def fit(self, rng_key, X, y, num_warmup, num_samples, num_chains, print_summary=True, **kw):
        log.append(np.asarray(rng_key).copy())
        rng = np.random.default_rng(len(log))
        a = rng.standard_normal((1, 100))
        if not rhat_ok(len(log)):
            a = a + np.linspace(0, 5, 100)           # drifting chain: split r-hat far above 1.1
        k = rng.standard_normal((1, 100, 2))
        mu = np.broadcast_to(np.linspace(0, 50, 100)[None, :, None], (1, 100, np.size(X)))   # drifts: r-hat skips it
        self.mcmc = MCMCResult({"a": a, "k": k, "noise": np.abs(rng.standard_normal((1, 100))) + 1, "mu": mu}, [{}])
    return fit


@pytest.mark.parametrize("good_from,restarts,fits", [(1, 3, 1), (2, 3, 2), (3, 3, 3), (99, 3, 3), (99, 1, 1)])
def test_restarts_refit_only_while_rhat_is_high(monkeypatch, good_from, restarts, fits):
    log = []
    monkeypatch.setattr(sPM, "fit", _fake_fit(log, lambda call: call >= good_from))
    X, y = get_dummy_data()
    _, m = step(model, model_priors, X, y, num_restarts=restarts, print_summary=False)
    assert len(log) == fits
    for i, key in enumerate(log):
        assert np.array_equal(key, get_keys(i)[0])


def test_vector_site_rhat_takes_the_largest_component(monkeypatch):
    """a vector site whose second component does not mix forces a restart (the reference raises on vector sites)"""
    log = []

    def fit(self, rng_key, X, y, *a, **kw):
        log.append(1)
        rng = np.random.default_rng(0)
        k = rng.standard_normal((1, 100, 2))
        k[0, :, 1] += np.linspace(0, 5, 100)
        self.mcmc = MCMCResult({"k": k, "noise": np.abs(rng.standard_normal((1, 100))) + 1}, [{}])
    monkeypatch.setattr(sPM, "fit", fit)
    X, y = get_dummy_data()
    step(model, model_priors, X, y, num_restarts=2, print_summary=False)
    assert len(log) == 2


# ---- the reference's tests/test_hypo.py, gp_wrap=False (gp_wrap=True is in test_gpu_hypo.py)
@pytest.mark.parametrize("method", ["softmax", "eps-greedy"])
def test_reference_sample_next(method):
    idx = sample_next(np.array([0.0, 0.1, 0.2]), method)
    assert isinstance(idx, (np.int64, int))


def test_reference_step_standalone():
    X, y = get_dummy_data()
    obj, _ = step(model, model_priors, X, y, X, gp_wrap=False, num_warmup=50, num_samples=50)
    assert isinstance(obj, np.ndarray) and obj.shape == X.shape
