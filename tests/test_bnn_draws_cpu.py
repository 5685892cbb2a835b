"""CPU: the host side of BNN's lock-step chains.  BNNLogJoint.batch against __call__ row by row (invalid noise rows kept
off the library), vectorized NUTS chains against sequential ones with one likelihood call per round, and
Context.bnn_loglik_draws' argument checks.  A stub context evaluates the NumPy oracle (oracle/bnn_oracle.py), the same
function for single and batched calls, so equal rows are equal bits."""
import numpy as np
import pytest

from oracle import bnn_oracle as bo


class _Dev:
    def __init__(self, a):
        self.a = a

    def free(self):
        pass


class _StubCtx:
    """stands in for _ffi.Context: the oracle's likelihood, one draw at a time or for a batch of weight sets"""

    def __init__(self):
        self.calls = {"bnn_loglik": 0, "bnn_loglik_draws": 0}
        self.sigmas = []

    def to_device(self, a):
        return _Dev(np.asarray(a))

    def bnn_loglik(self, Xd, yd, widths, act, flat, sigma):
        self.calls["bnn_loglik"] += 1
        v, gs, gp, _ = bo.loglik(Xd.a, yd.a, Xd.a.shape[1], list(widths), flat, sigma)
        return v, gs, gp

    def bnn_loglik_draws(self, Xd, yd, widths, act, params, sigma, want_params=True):
        self.calls["bnn_loglik_draws"] += 1
        sigma = np.asarray(sigma, dtype=np.float64)
        self.sigmas.append(sigma)
        assert params.ndim == 2 and params.shape[0] == sigma.size
        out = [bo.loglik(Xd.a, yd.a, Xd.a.shape[1], list(widths), p, float(s))[:3] for p, s in zip(params, sigma)]
        return np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.stack([o[2] for o in out])

    def bnn_predict(self, X, widths, act, params, sigma=None, eps=None):
        return bo.predict(np.asarray(X), np.asarray(X).shape[1], list(widths), params, sigma, eps)


def _log_joint(seed=3, noise_prior=None):
    from gpax_b200 import BNN
    from gpax_b200.bnn import BNNLogJoint
    ctx = _StubCtx()
    m = BNN(2, 2, noise_prior_dist=noise_prior, hidden_dim=[4, 3], ctx=ctx)
    rng = np.random.default_rng(seed)
    X, y = rng.uniform(-1, 1, (9, 2)), rng.standard_normal((9, 2))
    return BNNLogJoint(m, X, y, rng), ctx, rng


@pytest.mark.parametrize("noise_prior", [None, "halfnormal"])
def test_batch_rows_equal_single_calls_bit_for_bit(noise_prior):
    from gpax_b200 import priors as P
    lj, ctx, rng = _log_joint(noise_prior=P.HalfNormal(0.5) if noise_prior else None)
    u0 = lj.init_u()
    U = u0[None] + 0.2 * rng.standard_normal((6, u0.size))
    U[1, 0] = 1e6                     # the noise overflows to inf
    U[4, 0] = np.nan                  # no noise at all
    for jac in (False, True):
        n0 = lj.n_evals
        vals, grads = lj.batch(U, jac)
        assert lj.n_evals == n0 + len(U)
        assert ctx.calls["bnn_loglik_draws"] == (1 if not jac else 2)
        # the invalid rows never reach the library
        assert ctx.sigmas[-1].size == 4 and np.all(np.isfinite(ctx.sigmas[-1])) and np.all(ctx.sigmas[-1] > 0)
        single = ctx.calls["bnn_loglik"]
        for r, u in enumerate(U):
            v, g = lj(u, jac)
            assert vals[r] == v or (np.isnan(v) and np.isnan(vals[r])), r
            assert np.array_equal(grads[r], g), r
        assert ctx.calls["bnn_loglik"] == single + 4
        assert vals[1] == -np.inf and vals[4] == -np.inf and not grads[[1, 4]].any()
        assert np.isfinite(vals[[0, 2, 3, 5]]).all()


def test_batch_of_only_invalid_rows_makes_no_library_call():
    lj, ctx, rng = _log_joint()
    U = np.tile(lj.init_u(), (3, 1))
    U[:, 0] = [1e6, np.nan, np.inf]
    vals, grads = lj.batch(U, True)
    assert ctx.calls == {"bnn_loglik": 0, "bnn_loglik_draws": 0}
    assert np.all(vals == -np.inf) and not grads.any() and grads.shape == (3, lj.dim)


def test_vectorized_chains_equal_sequential_with_one_call_per_round():
    from gpax_b200 import BNN
    X = np.linspace(-1, 1, 12)
    y = np.sin(2 * X)
    runs = {}
    for method in ("sequential", "vectorized"):
        ctx = _StubCtx()
        m = BNN(1, 1, hidden_dim=[3], ctx=ctx)
        m.fit(0, X, y, num_warmup=15, num_samples=10, num_chains=3, chain_method=method, progress_bar=False,
              print_summary=False)
        runs[method] = (m.get_samples(chain_dim=True), m.mcmc.stats, dict(ctx.calls))
    (s_seq, st_seq, c_seq), (s_vec, st_vec, c_vec) = runs["sequential"], runs["vectorized"]
    assert list(s_seq) == list(s_vec)
    for k in s_seq:
        assert s_seq[k].shape[:2] == (3, 10) and np.array_equal(s_seq[k], s_vec[k]), k
    assert st_seq == st_vec
    rounds = max(np.diff([0] + [s["grad_evals"] for s in st_vec]))
    assert c_vec == {"bnn_loglik": 0, "bnn_loglik_draws": rounds}
    assert c_seq["bnn_loglik_draws"] == 0 and c_seq["bnn_loglik"] == st_seq[-1]["grad_evals"]


def test_draws_binding_checks_shapes_before_calling_the_library():
    """nothing of the context is touched before the checks, so a bare instance shows them"""
    from gpax_b200 import _ffi
    ctx = object.__new__(_ffi.Context)
    X, y, widths = np.ones((4, 2)), np.ones((4, 1)), [3, 1]
    good = np.zeros((2, 2 * 3 + 3 + 3 + 1))
    with pytest.raises(ValueError):
        ctx.bnn_loglik_draws(X, y, widths, 1, good[:, :-1], [0.1, 0.1])     # rows for another network
    with pytest.raises(ValueError):
        ctx.bnn_loglik_draws(X, y, widths, 1, good[0], [0.1])                # one flat vector, not [S, P]
    with pytest.raises(ValueError):
        ctx.bnn_loglik_draws(X, y, widths, 1, good, [0.1, 0.1, 0.1])         # sigma for another S
    with pytest.raises(ValueError):
        ctx.bnn_loglik_draws(X, np.ones((4, 2)), widths, 1, good, [0.1, 0.1])
    with pytest.raises(ValueError):
        ctx.bnn_loglik_draws(np.ones((4, 1)), y, widths, 1, good, [0.1, 0.1])
