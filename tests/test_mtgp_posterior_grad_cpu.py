"""CPU: the derivative behind optimize_acq on MultiTaskGP / CoregGP, pinned by central differences (no JAX here to pin it
to).

- mtgp_grad_oracle.posterior_grad's d mean / dx and d var / dx against central differences of
  oracle.mtgp_oracle.posterior, for the three kernels, L in {1, 2} latents, T in {2, 3} tasks, d in {1, 3}, noiseless
  both ways and both forms.  In the multitask form that includes the task column, whose difference is exactly 0 away
  from an integer;
- which multi-task models and acquisitions acquisition.optimize_acq differentiates in closed form."""
import itertools

import numpy as np
import pytest

from gpax_b200 import acquisition as acq
from mtgp_grad_oracle import posterior_grad
from oracle import mtgp_oracle as mo

H = 1e-5


def problem(kernel, L, T, d, shared, seed=0, n=10, P=3):
    rng = np.random.default_rng(seed + 100 * L + 10 * T + d + 1000 * shared)
    p = {"k_length": rng.uniform(0.5, 0.9, (L, d)), "k_scale": rng.uniform(0.8, 1.3, L), "W": rng.normal(0, 0.7, (L, T, 2)),
         "v": rng.uniform(0.3, 0.8, (L, T)), "noise": rng.uniform(0.05, 0.2, T),
         "period": rng.uniform(1.5, 2.5, L) if kernel == "Periodic" else None}
    X = rng.uniform(0, 2, (n, d))
    Xn = rng.uniform(0, 2, (P, d))
    if not shared:
        X = np.c_[X, rng.integers(0, T, n)]
        Xn = np.c_[Xn, rng.integers(0, T, P) + 0.4]         # off the integers: astype(int) is locally constant
    y = rng.standard_normal(n * T if shared else n)
    return X, y, Xn, p


CASES = list(itertools.product(["RBF", "Matern", "Periodic"], [1, 2], [2, 3], [1, 3], [False, True], [False, True]))


@pytest.mark.parametrize("kernel,L,T,d,noiseless,shared", CASES)
def test_oracle_gradient_vs_central_differences(kernel, L, T, d, noiseless, shared):
    X, y, Xn, p = problem(kernel, L, T, d, shared)
    mean, var, dmean, dvar = posterior_grad(X, y, Xn, p, kernel, shared, T, noiseless)
    group = T if shared else 1
    P, cols = Xn.shape
    assert dmean.shape == dvar.shape == (P * group, cols)
    for i in range(P):
        for k in range(cols):
            e = np.zeros_like(Xn)
            e[i, k] = H
            mp, cp = mo.posterior(X, y, Xn + e, p, kernel, shared, T, noiseless)
            mm, cm = mo.posterior(X, y, Xn - e, p, kernel, shared, T, noiseless)
            rows = slice(i * group, (i + 1) * group)                # the GP rows of point i
            fd_m = (mp - mm)[rows] / (2 * H)
            fd_v = (np.diag(cp) - np.diag(cm))[rows] / (2 * H)
            if not shared and k == cols - 1:
                assert np.all(fd_m == 0) and np.all(fd_v == 0)
                assert np.all(dmean[rows, k] == 0) and np.all(dvar[rows, k] == 0)
                continue
            np.testing.assert_allclose(dmean[rows, k], fd_m, rtol=1e-6, atol=1e-7 * max(1.0, np.abs(dmean).max()))
            np.testing.assert_allclose(dvar[rows, k], fd_v, rtol=1e-6, atol=1e-7 * max(1.0, np.abs(dvar).max()))
    m0, c0 = mo.posterior(X, y, Xn, p, kernel, shared, T, noiseless)
    np.testing.assert_array_equal(mean, m0)
    np.testing.assert_array_equal(var, np.diag(c0))


def test_optimize_acq_differentiates_multitask_form_lcm_models():
    from gpax_b200 import CoregGP, MultiTaskGP
    mt = MultiTaskGP(2, "RBF", num_latents=2, num_tasks=2)
    cg = CoregGP(2, "Matern")
    for model in (mt, cg):
        assert acq._analytic_kind(acq.EI, model, {}) == "EI", type(model).__name__
        assert acq._analytic_kind(acq.UCB, model, {}) == "UCB"
        assert acq._analytic_kind(acq.POI, model, {}) == "POI"
        assert acq._analytic_kind(acq.UE, model, {}) == "UE"
        assert acq._analytic_kind(acq.EI, model, {"penalty": "delta"}) is None
        assert acq._analytic_kind(acq.KG, model, {}) is None
        assert acq._analytic_kind(acq.Thompson, model, {}) is None
    assert acq._analytic_kind(acq.EI, MultiTaskGP(2, "RBF", shared_input_space=True, num_tasks=2), {}) is None
    assert acq._analytic_kind(acq.EI, MultiTaskGP(2, "RBF", num_latents=2, num_tasks=2, mean_fn=lambda x: 0.0 * x[:, 0]), {}) is None
    assert acq._analytic_kind(acq.EI, CoregGP(2, "RBF", mean_fn=lambda x: 0.0 * x[:, 0]), {}) is None

    class MyMTGP(MultiTaskGP):
        pass
    assert acq._analytic_kind(acq.EI, MyMTGP(2, "RBF", num_latents=2, num_tasks=2), {}) is None


def test_posterior_grad_refuses_the_kronecker_form_and_mean_functions():
    from gpax_b200 import MultiTaskGP
    kron = MultiTaskGP(1, "RBF", shared_input_space=True, num_tasks=2)
    kron.X_train, kron.y_train = np.zeros((3, 1)), np.zeros(6)
    with pytest.raises(NotImplementedError):
        kron._posterior_grad(np.zeros((1, 1)), {}, True, False)
    mf = MultiTaskGP(1, "RBF", num_latents=1, num_tasks=2, mean_fn=lambda x: 0.0 * x[:, 0])
    mf.X_train, mf.y_train = np.c_[np.zeros(3), [0, 1, 0]], np.zeros(3)
    with pytest.raises(NotImplementedError):
        mf._posterior_grad(np.zeros((1, 2)), {}, True, False)
