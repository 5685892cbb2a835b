"""CPU: viSparseGP with a user kernel callable -- the Gram-block oracle of the VFE bound and the sparse posterior
(tests/sparse_gram_oracle.py) against the existing closed-form oracle and the reference's golden vectors, and the host
side of SparseGramLogJoint (kernel calls, Xu shifts, chunked diagonal, chain rule) run against the oracle in place of
the library."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle  # noqa: E402
from oracle import fit_oracle as fo  # noqa: E402
import sparse_gram_oracle as so  # noqa: E402
from gpax_b200 import inference, priors  # noqa: E402
from gpax_b200.sparse_gp import viSparseGP  # noqa: E402
from gpax_b200.utils import set_kernel_fn  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_vectors_sparse_callable.npz")


def _exact_dirs(kind, Xu, X, theta, jitter):
    """blocks and exact d/dlog(theta) directions of the built-in kernel (fit_oracle's derivatives)"""
    M = Xu.shape[0]
    k, dK = fo._derivs(np.vstack([Xu, X]), theta, kind)
    blocks = (k[:M, :M] + jitter * np.eye(M), k[:M, M:], np.diag(k)[M:].copy())
    idx = [p for p in range(len(dK)) if dK[p] is not None]
    dirs = [(dK[p][:M, :M], dK[p][:M, M:], np.diag(dK[p])[M:].copy()) for p in idx]
    return blocks, dirs, idx


@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
@pytest.mark.parametrize("clip", [False, True])
def test_gram_oracle_matches_closed_form_oracle(kind, clip):
    Xu, X, y, theta = fo.elbo_problem(kind, 9, 37, 2, seed=3)
    if clip:          # the inducing points on the data: T = 0 up to rounding, both sides of the clip are exercised
        Xu = X[:9].copy()
    jitter = 1e-6
    v0, g0, gx0, _, _, _ = fo.elbo_grad(kind, Xu, X, y, theta, jitter)
    blocks, dirs, idx = _exact_dirs(kind, Xu, X, theta, jitter)
    v, g, gln, _, alpha = so.elbo_gram_grad(*blocks, y, theta[2 + 1], dirs)
    np.testing.assert_allclose(v, v0, rtol=1e-12)
    np.testing.assert_allclose(g, g0[idx], rtol=1e-9, atol=1e-9 * np.abs(g0).max())
    np.testing.assert_allclose(gln, g0[2 + 1], rtol=1e-9, atol=1e-12)
    # alpha = d value / d mean: a central difference of the bound in the direction of a mean vector
    dm = np.cos(np.arange(X.shape[0]))
    h = 1e-6
    fd = (so.elbo_gram_grad(*blocks, y - h * dm, theta[3])[0] - so.elbo_gram_grad(*blocks, y + h * dm, theta[3])[0]) / (2 * h)
    assert abs(fd - alpha @ dm) <= 1e-6 * max(1.0, abs(fd))


def _golden_kernels(z, tag):
    if tag == "linrbf":
        def linrbf(X, Z, k_scale, k_length, c):
            r2 = (((X[:, None, :] - Z[None, :, :]) / k_length) ** 2).sum(-1)
            return k_scale * np.exp(-0.5 * r2) + c * X @ Z.T
        return set_kernel_fn(linrbf)
    return oracle.rbf_kernel


@pytest.mark.parametrize("tag", ["linrbf", "rbf"])
def test_gram_posterior_oracle_matches_reference(tag):
    z = np.load(GOLDEN)
    X, y, Xu, Xs = z[tag + "_Xtr"], z[tag + "_ytr"], z[tag + "_Xu"], z[tag + "_Xte"]
    params = {k[len(tag) + 3:]: z[k] for k in z.files if k.startswith(tag + "_p_")}
    k = _golden_kernels(z, tag)
    for key, nl, kw in (("nl0", False, {}), ("nl1", True, {}), ("jit1e-5", False, {"jitter": 1e-5})):
        noise = float(params["noise"])
        Kuu = k(Xu, Xu, params, **kw)
        Kss = k(Xs, Xs, params, noise * (1 - int(nl)), **kw)
        mean, cov = so.sparse_posterior_gram(Kuu, k(Xu, X, params, jitter=0), y, noise, k(Xu, Xs, params, jitter=0), Kss)
        np.testing.assert_allclose(mean, z[f"{tag}_{key}_mean"], rtol=1e-9, atol=1e-10)
        np.testing.assert_allclose(cov, z[f"{tag}_{key}_cov"], rtol=1e-9, atol=1e-10)


class _OracleCtx:
    """stands in for the library: sparse_elbo_gram from the oracle"""

    def __init__(self):
        self.calls = []

    def sparse_elbo_gram(self, Kuu, Kuf, kff_diag, yres, noise, dirs=(), rdirs=(), want_alpha=False):
        self.calls.append((len(dirs), len(rdirs)))
        v, g, gln, rows, alpha = so.elbo_gram_grad(Kuu, Kuf, kff_diag, yres, noise, dirs, rdirs)
        return {"value": v, "grad": g, "grad_log_noise": gln, "grad_rows": rows, "alpha": alpha if want_alpha else None,
                "info": 0}


def _sparse_model(kernel, d, N, seed, mean=False):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (N, d))
    y = np.sin(2 * X[:, 0]) + 0.5 * X[:, -1] + 0.05 * rng.standard_normal(N)
    kw = {}
    if mean:
        kw = {"mean_fn": lambda x, p: p["a"] * x[:, 0] + p["b"],
              "mean_fn_prior": lambda: {"a": priors.sample("a", priors.Normal(0.0, 1.0)),
                                        "b": priors.sample("b", priors.Normal(0.0, 1.0))}}
    m = viSparseGP(d, kernel, ctx=_OracleCtx(), **kw)
    m.X_train, m.y_train = X, y
    return m, X, y


def test_xu_shift_directions_give_the_bound_gradient():
    """grad_rows from the Xu-shifted blocks against the analytic d value / d Xu of the closed-form oracle"""
    kind, d = "RBF", 2
    Xu, X, y, theta = fo.elbo_problem(kind, 8, 41, d, seed=5)
    m, _, _ = _sparse_model(oracle.rbf_kernel, d, 41, 0)
    m.X_train, m.y_train = X, y
    lj = inference.SparseGramLogJoint(m, Xu, jitter=1e-6)
    kp = {"k_length": theta[:d], "k_scale": theta[d], "period": None}
    blocks = lj._blocks(kp)
    _, _, _, rows, _ = so.elbo_gram_grad(*blocks, y, theta[d + 1], (), lj._xu_dirs(kp))
    _, _, gx0, _, _, _ = fo.elbo_grad(kind, Xu, X, y, theta, 1e-6)
    np.testing.assert_allclose(rows.T, gx0, rtol=1e-6, atol=1e-7 * np.abs(gx0).max())


def test_kff_diagonal_from_chunks_matches_the_full_call():
    m, X, _ = _sparse_model(oracle.matern_kernel, 3, 53, 1)
    lj = inference.SparseGramLogJoint(m, X[:7], jitter=1e-6)
    kp = {"k_length": np.array([0.4, 0.5, 0.6]), "k_scale": 1.3, "period": None}
    lj.KFF_CHUNK = 10
    Kuu, Kuf, kff = lj._blocks(kp)
    np.testing.assert_array_equal(kff, np.diag(oracle.matern_kernel(X, X, kp, jitter=0)))
    np.testing.assert_array_equal(Kuu, oracle.matern_kernel(X[:7], X[:7], kp, jitter=1e-6))
    np.testing.assert_array_equal(Kuf, oracle.matern_kernel(X[:7], X, kp))


def test_kuf_keeps_the_reference_shape_rule_when_m_equals_n():
    """Kuf = k(Xu, X, params) with the callable's default jitter: on its diagonal when M == N (sparse_gp.py:96)"""
    m, X, _ = _sparse_model(oracle.rbf_kernel, 1, 6, 2)
    lj = inference.SparseGramLogJoint(m, X[::-1].copy(), jitter=1e-6)
    kp = {"k_length": np.array([0.5]), "k_scale": 1.0, "period": None}
    _, Kuf, _ = lj._blocks(kp)
    np.testing.assert_array_equal(Kuf, oracle.rbf_kernel(X[::-1], X, kp, 0, 1e-6))
    assert not np.array_equal(Kuf, oracle.rbf_kernel(X[::-1], X, kp, 0, 0.0))


@pytest.mark.parametrize("mean", [False, True])
def test_log_joint_gradient_matches_differences_of_the_oracle(mean):
    """the whole host chain rule (kernel sites, noise, mean_fn_prior sites, priors) against central differences of the
    log joint it evaluates; grad_Xu against differences in Xu"""
    m, X, y = _sparse_model(oracle.rbf_kernel, 2, 33, 3, mean=mean)
    lj = inference.SparseGramLogJoint(m, X[:6] + 0.01, jitter=1e-6)
    u = lj.init_u() + 0.1 * np.arange(lj.dim)
    val, g = lj(u, jacobian=True)
    gx = lj.grad_Xu.copy()
    h = 1e-5
    fd = np.array([(lj(u + h * e, True)[0] - lj(u - h * e, True)[0]) / (2 * h) for e in np.eye(lj.dim)])
    np.testing.assert_allclose(g, fd, rtol=1e-5, atol=1e-6)
    Xu0 = lj.Xu.copy()
    for a, k in ((0, 0), (3, 1)):
        E = np.zeros_like(Xu0)
        E[a, k] = h
        lj.Xu = Xu0 + E
        vp = lj(u, True)[0]
        lj.Xu = Xu0 - E
        vm = lj(u, True)[0]
        assert abs((vp - vm) / (2 * h) - gx[a, k]) <= 1e-5 * max(1.0, abs(gx[a, k]))
    lj.Xu = Xu0
    # one library call per evaluation: the kernel directions (k_length[2], k_scale) and the d Xu directions
    assert m.ctx.calls[0] == (3, 2)
    assert math.isfinite(val)


def test_fit_dispatch(monkeypatch):
    """a callable picks SparseGramLogJoint; the fused kernels keep their log joints, and a probabilistic mean function
    on a fused kernel is no longer refused"""
    made = []

    class Spy(inference.SparseGramLogJoint):
        def __init__(self, *a, **k):
            made.append(type(self))
            super().__init__(*a, **k)
    monkeypatch.setattr(inference, "SparseGramLogJoint", Spy)
    monkeypatch.setattr(inference, "adam", lambda params, objective, *a: (params, []))
    m, X, _ = _sparse_model(oracle.rbf_kernel, 2, 20, 4)
    inference.fit_sparse_gp(m, 0, X[:4], 1, 1e-3, False)
    assert made == [Spy]
    f, _, _ = _sparse_model("RBF", 2, 20, 4, mean=True)
    lj = inference._sparse_program_log_joint(f, X[:4], 1e-6)
    assert lj.has_mean_params and not isinstance(lj, inference.SparseGramLogJoint)
