"""CPU: the host logic of the acquisition functions on a BNN.

- which acquisitions optimize_acq differentiates in closed form on a BNN (one vs two outputs, with and without a
  penalty, each acquisition function);
- the draw count Thompson sampling takes from the samples' first site, on GP and BNN samples, and the layout a BNN's
  Thompson sample comes back in (a BNN whose predict is replaced, so no device is needed);
- the refusals: two-output and unfitted BNNs, KG / qKG, and noiseless q-batch acquisitions."""
import numpy as np
import pytest

from gpax_b200 import BNN, prng
from gpax_b200 import acquisition as acq

S, P = 6, 5


def _samples(hidden=(4,), D=1, O=1, seed=0):
    rng = np.random.default_rng(seed)
    out, i = {}, D
    for l, w in enumerate(list(hidden) + [O]):
        out[f"w{l}"] = rng.standard_normal((S, i, w))
        out[f"b{l}"] = rng.standard_normal((S, w))
        i = w
    out["noise"] = rng.uniform(0.1, 0.2, S)
    out["mu"] = rng.standard_normal((S, 3, O))
    return out


class _FittedBNN(BNN):
    """a BNN with posterior samples and a host-side predict that records its calls"""

    def __init__(self, O=1):
        super().__init__(1, O, hidden_dim=[4])
        self.mcmc = object()
        self.samples = _samples(O=O)
        self.calls = []

    def get_samples(self, chain_dim=False):
        return self.samples

    def predict(self, rng_key, X_new, samples=None, n=1, **kwargs):
        samples = self.samples if samples is None else samples
        self.calls.append((samples, n, kwargs))
        k = len(samples["noise"])
        loc = np.arange(k * P, dtype=np.float64).reshape(k, P, 1)
        return loc.mean(0), loc + 0.5


@pytest.mark.parametrize("fn,kind", [(acq.EI, "EI"), (acq.UCB, "UCB"), (acq.POI, "POI"), (acq.UE, "UE")])
def test_analytic_kind_admits_one_output_bnns_without_a_penalty(fn, kind):
    assert acq._analytic_kind(fn, BNN(1, 1), {}) == kind
    assert acq._analytic_kind(fn, BNN(3, 1, hidden_dim=[16, 8, 4]), {"noiseless": True}) == kind
    assert acq._analytic_kind(fn, BNN(1, 2), {}) is None
    assert acq._analytic_kind(fn, BNN(1, 1), {"penalty": "delta", "recent_points": np.zeros((1, 1))}) is None


@pytest.mark.parametrize("fn", [acq.KG, acq.Thompson, acq.qEI, acq.qUCB, acq.qPOI, acq.qKG])
def test_analytic_kind_leaves_the_other_acquisitions_on_finite_differences(fn):
    assert acq._analytic_kind(fn, BNN(1, 1), {}) is None


def test_analytic_kind_refuses_bnn_subclasses():
    class MyBNN(BNN):
        pass
    assert acq._analytic_kind(acq.EI, MyBNN(1, 1), {}) is None


def test_draw_count_from_the_first_site():
    gp = {"k_length": np.ones((7, 2)), "k_scale": np.ones(7), "noise": np.ones(7)}
    assert acq._num_draws(gp) == len(gp["k_length"]) == 7
    assert acq._num_draws(_samples()) == S


@pytest.mark.parametrize("n", [1, 3])
def test_thompson_on_a_bnn_picks_the_draw_and_returns_the_gp_layout(n):
    m = _FittedBNN()
    X = np.linspace(-1, 1, P)
    got = acq.Thompson(11, m, X, n=n, noiseless=True)
    idx = prng.randint(prng.as_key(11), (1,), 0, S)
    (samples, n_seen, kw), = m.calls
    assert n_seen == n and kw == {"noiseless": True}
    for k, v in m.samples.items():
        assert np.array_equal(samples[k], v[idx])
    row = np.arange(P, dtype=np.float64) + 0.5
    if n == 1:
        assert got.shape == (1, 1, P) and np.array_equal(got[0, 0], row)
    else:
        assert got.shape == (P,) and np.array_equal(got, row)


@pytest.mark.parametrize("fn", [acq.EI, acq.UCB, acq.POI, acq.UE, acq.Thompson, acq.qEI, acq.qUCB, acq.qPOI])
def test_two_output_bnn_is_refused(fn):
    m = _FittedBNN(O=2)
    with pytest.raises(ValueError, match="one-output"):
        fn(0, m, np.zeros((3, 1)))
    assert m.calls == []


@pytest.mark.parametrize("fn", [acq.EI, acq.UCB, acq.POI, acq.UE, acq.Thompson, acq.qEI])
def test_unfitted_bnn_is_refused(fn):
    with pytest.raises(ValueError, match="fit it first"):
        fn(0, BNN(1, 1), np.zeros((3, 1)))


@pytest.mark.parametrize("fn", [acq.KG, acq.qKG])
def test_kg_is_refused_on_a_bnn(fn):
    m = _FittedBNN()
    with pytest.raises(ValueError, match="refit"):
        fn(0, m, np.zeros((3, 1)))
    assert m.calls == []


@pytest.mark.parametrize("fn", [acq.qEI, acq.qUCB, acq.qPOI])
def test_noiseless_q_batch_is_refused_on_a_bnn(fn):
    with pytest.raises(ValueError, match="noiseless=False"):
        fn(0, _FittedBNN(), np.zeros((3, 1)), noiseless=True)
