"""CPU: run_nuts' chain methods on NumPy log joints.  "vectorized" advances the chains in lock-step rounds (one `batch`
call per round when the log joint has one) and must give the draws and stats of "sequential" bit for bit."""
import numpy as np
import pytest

from gpax_b200 import inference as inf


class Gauss:
    """a correlated Gaussian, log N(u; mu, S) with the LogJoint interface"""

    def __init__(self):
        self.mu = np.array([0.5, -1.0, 2.0])
        A = np.array([[1.0, 0.0, 0.0], [0.8, 0.6, 0.0], [-0.3, 0.4, 0.5]])
        self.P = np.linalg.inv(A @ A.T)
        self.dim, self.n_evals = 3, 0

    def init_u(self):
        return np.zeros(self.dim)

    def __call__(self, u, jacobian):
        self.n_evals += 1
        z = u - self.mu
        g = -self.P @ z
        return float(0.5 * z @ g), g

    def to_dict(self, U):
        return {"u": np.atleast_2d(U).copy()}


class Funnel(Gauss):
    """Neal's funnel in 3 dimensions: v ~ N(0, 1.5^2), x_k | v ~ N(0, exp(v))"""

    def __init__(self):
        self.dim, self.n_evals = 3, 0

    def __call__(self, u, jacobian):
        self.n_evals += 1
        v, x = u[0], u[1:]
        val = -0.5 * v * v / 2.25 - 0.5 * np.sum(x * x) * np.exp(-v) - 0.5 * v * x.size
        g = np.empty(3)
        g[0] = -v / 2.25 + 0.5 * np.sum(x * x) * np.exp(-v) - 0.5 * x.size
        g[1:] = -x * np.exp(-v)
        return float(val), g


def with_batch(cls):
    """the toy with a `batch` that evaluates the rows one by one and records the number of rows of every call"""

    class Batched(cls):
        def __init__(self):
            super().__init__()
            self.calls = []

        def batch(self, U, jacobian):
            self.calls.append(len(U))
            out = [cls.__call__(self, u, jacobian) for u in U]
            return np.array([o[0] for o in out]), np.stack([o[1] for o in out])

    return Batched


TOYS = {"gauss": Gauss, "funnel": Funnel, "gauss_batch": with_batch(Gauss), "funnel_batch": with_batch(Funnel)}
WARMUP, SAMPLES = 60, 30    # >= 40 warm-up draws: the diagonal metric is installed at 3/4 of warm-up


@pytest.mark.parametrize("toy", sorted(TOYS))
@pytest.mark.parametrize("chains", [1, 3, 5])
def test_vectorized_chains_match_sequential_bit_for_bit(toy, chains):
    seq_lj, vec_lj = TOYS[toy](), TOYS[toy]()
    seq = inf.run_nuts(seq_lj, 7, WARMUP, SAMPLES, chains, False, chain_method="sequential")
    vec = inf.run_nuts(vec_lj, 7, WARMUP, SAMPLES, chains, False, chain_method="vectorized")
    a, b = seq.get_samples(group_by_chain=True)["u"], vec.get_samples(group_by_chain=True)["u"]
    assert a.shape == (chains, SAMPLES, 3)
    assert np.array_equal(a, b)
    assert seq.stats == vec.stats
    # grad_evals is cumulative over chains 0..c, as when the chains ran one after another
    assert all(s1["grad_evals"] < s2["grad_evals"] for s1, s2 in zip(seq.stats, seq.stats[1:]))
    assert seq.stats[-1]["grad_evals"] == seq_lj.n_evals == vec_lj.n_evals
    if chains > 1:     # the chains are distinct (own seeds, jittered starts)
        assert not np.array_equal(a[0], a[1])


@pytest.mark.parametrize("toy", ["gauss_batch", "funnel_batch"])
def test_vectorized_makes_one_batch_call_per_round(toy):
    chains = 4
    lj = TOYS[toy]()
    res = inf.run_nuts(lj, 3, WARMUP, SAMPLES, chains, False, chain_method="vectorized")
    assert lj.calls and max(lj.calls) <= chains and min(lj.calls) >= 1
    # every round is one call; a round has one row per unfinished chain, so the rows add up to all evaluations
    assert sum(lj.calls) == res.stats[-1]["grad_evals"]
    # rounds = the longest chain's evaluations, since every unfinished chain evaluates once per round
    own = np.diff([0] + [s["grad_evals"] for s in res.stats])
    assert len(lj.calls) == max(own)
    assert lj.calls == sorted(lj.calls, reverse=True)     # chains only ever leave the rounds


def test_sequential_never_calls_batch_and_other_methods_run_sequentially():
    lj = TOYS["gauss_batch"]()
    ref = inf.run_nuts(TOYS["gauss"](), 11, WARMUP, SAMPLES, 2, False)
    for method in ("sequential", "parallel", "no-such-method"):
        got = inf.run_nuts(lj, 11, WARMUP, SAMPLES, 2, False, chain_method=method)
        assert np.array_equal(got.get_samples()["u"], ref.get_samples()["u"])
    assert lj.calls == []


def test_adaptation_is_reached_in_every_chain():
    res = inf.run_nuts(TOYS["gauss_batch"](), 5, 200, 200, 3, False, chain_method="vectorized")
    u = res.get_samples(group_by_chain=True)["u"]
    for c in range(3):
        assert 0.05 < res.stats[c]["step_size"] < 3.0
        np.testing.assert_allclose(u[c].mean(0), Gauss().mu, atol=0.6)


def test_old_entry_points_drive_the_generators():
    lj = Gauss()
    rng = np.random.default_rng(0)
    u = np.zeros(3)
    lp, g = lj(u, True)
    eps = inf._find_eps(lj, u, lp, g, rng, np.ones(3))
    u2, lp2, g2, acc, depth, div = inf._nuts_draw(lj, u, lp, g, eps, rng, np.ones(3))
    assert eps > 0 and u2.shape == (3,) and 0.0 <= acc <= 1.0 and np.isfinite(lp2)
