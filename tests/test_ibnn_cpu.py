"""CPU checks of iBNN / vi_iBNN: the oracle's likelihood gradient against central differences (the GPU gradient is tested
against this oracle), the site names, default priors and theta packing of both log joints, depth 0, and the routing of
the acquisition optimiser."""
import numpy as np
import pytest

from gpax_b200 import acquisition, iBNN, vi_iBNN
from gpax_b200 import priors as P
from gpax_b200.ibnn import nngp_theta_rows
from gpax_b200.inference import NNGPLogJoint, ProgramLogJoint, make_log_joint
from oracle import ibnn_oracle as io


def _data(N=8, d=1, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (N, d))
    return X, 10 * X[:, 0] ** 2            # the reference's own test data shape (tests/test_ibnn.py)


def _params(th, d):
    return {"var_w": th[d], "noise": th[d + 1], "var_b": th[d + 2]}


def cpu_lik(model, X):
    """the likelihood of b2gp_mll on the host: value, grad [d+3] in its layout, info"""
    d = X.shape[1]

    def lik(th, yres):
        v, g = io.mll_grad(X, yres, _params(th, d), model.activation, int(th[0]))
        full = np.zeros(d + 3)
        full[d:] = g
        return v, full, None, 0
    return lik


@pytest.mark.parametrize("d", [1, 5, 40])
@pytest.mark.parametrize("depth", [0, 1, 2, 3])
@pytest.mark.parametrize("act", ["erf", "relu"])
def test_oracle_gradient_matches_central_differences(act, depth, d):
    rng = np.random.default_rng(depth * 100 + d)
    X = rng.uniform(-1, 1, (30, d))
    X[3] = X[7]                                          # a duplicated input
    y = rng.standard_normal(30)
    p = {"var_b": 0.7, "var_w": 1.6, "noise": 0.05}
    v, g = io.mll_grad(X, y, p, act, depth)
    assert abs(v - io.mll(X, y, p, act, depth)) < 1e-10 * abs(v)
    h, fd = 1e-5, []
    for name in ("var_w", "noise", "var_b"):
        pp, pm = dict(p), dict(p)
        pp[name], pm[name] = p[name] * np.exp(h), p[name] * np.exp(-h)
        fd.append((io.mll(X, y, pp, act, depth) - io.mll(X, y, pm, act, depth)) / (2 * h))
    np.testing.assert_allclose(g, fd, rtol=2e-6, atol=1e-6 * np.abs(g).max())


def test_relu_self_terms_sit_on_the_clip():
    X = np.random.default_rng(1).uniform(-1, 1, (6, 3))
    K, dKb, dKw = io.kernel_grad(X, X, 0.7, 1.6, "relu", 2)
    np.testing.assert_allclose(K, io.kernel(X, X, {"var_b": 0.7, "var_w": 1.6}, 0.0, 0.0, "relu", 2), rtol=1e-14)
    k0 = 0.7 + 1.6 * (X * X).sum(1) / 3
    assert np.all(k0 / np.sqrt(k0 * k0) == 1.0)          # a / sqrt(a a) = 1: above the clip, theta is constant there
    for i in range(6):                                   # the diagonal: d k11 / d var_b by differences of the self-chain
        h = 1e-6
        kp = io.kernel(X[i:i + 1], X[i:i + 1], {"var_b": 0.7 + h, "var_w": 1.6}, 0.0, 0.0, "relu", 2)[0, 0]
        km = io.kernel(X[i:i + 1], X[i:i + 1], {"var_b": 0.7 - h, "var_w": 1.6}, 0.0, 0.0, "relu", 2)[0, 0]
        assert abs(dKb[i, i] - (kp - km) / (2 * h)) < 1e-7


def test_theta_packing():
    th = nngp_theta_rows({"var_b": 0.3, "var_w": 2.0, "noise": 0.1}, 4, 3, False)
    np.testing.assert_array_equal(th, [[3, 3, 3, 3, 2.0, 0.1, 0.3]])
    th = nngp_theta_rows({"var_b": np.array([0.3, 0.4]), "var_w": np.array([2.0, 2.5]), "noise": np.array([0.1, 0.2])}, 1, 0, True)
    np.testing.assert_array_equal(th, [[0, 2.0, 0.1, 0.3], [0, 2.5, 0.2, 0.4]])
    m = vi_iBNN(2, depth=5, activation="relu")
    np.testing.assert_array_equal(m._theta({"var_b": 1.0, "var_w": 2.0, "noise": 3.0}, 2, False), [[5, 5, 2, 3, 1]])
    assert m._fused == "NNGP_relu" and iBNN(1)._fused == "NNGP_erf" and iBNN(1).depth == 3
    with pytest.raises(ValueError):
        iBNN(1, depth=17)


@pytest.mark.parametrize("cls", [iBNN, vi_iBNN])
@pytest.mark.parametrize("depth", [0, 2])
def test_log_joint_sites_priors_and_depth(cls, depth):
    X, y = _data()
    m = cls(1, depth=depth, activation="relu")
    m.X_train, m.y_train = X, y

    class CpuLJ(NNGPLogJoint):
        def _lik(self, th):
            v, g, _, info = cpu_lik(m, X)(th, self.y)
            return v, g, info
    lj = CpuLJ(m)
    assert isinstance(make_log_joint(m), NNGPLogJoint)
    assert lj.names == ["var_b", "var_w", "noise"]
    pb, pw, pn = lj.priors
    if cls is iBNN:                                      # ibnn.py:59-60, gp.py:222-227
        assert (type(pb), pb.loc, pb.scale, type(pw), pw.loc, pw.scale) == (P.LogNormal, 0.0, 1.0, P.LogNormal, 0.0, 1.0)
    else:                                                # vi_ibnn.py:58-59
        assert (type(pb), pb.scale, type(pw), pw.loc, pw.scale) == (P.HalfNormal, 1.0, P.LogNormal, 0.0, 10.0)
    assert (type(pn), pn.loc, pn.scale) == (P.LogNormal, 0.0, 1.0)
    u = np.array([-0.3, 0.2, -1.5])
    th = lj.theta_of(u)
    np.testing.assert_array_equal(th[:1], [depth])
    for jac in (False, True):
        v, g = lj(u, jac)
        assert np.isfinite(v) and np.all(np.isfinite(g))
        h, fd = 1e-6, np.zeros(3)
        for k in range(3):
            e = np.zeros(3)
            e[k] = h
            fd[k] = (lj(u + e, jac)[0] - lj(u - e, jac)[0]) / (2 * h)
        np.testing.assert_allclose(g, fd, rtol=1e-6, atol=1e-7)
    d = lj.to_dict(np.stack([u, u]))
    assert set(d) == {"var_b", "var_w", "noise"} and d["var_b"].shape == (2,)
    # the same model with the default sites restated as a prior program: ProgramLogJoint agrees, depth 0 included
    m2 = cls(1, depth=depth, activation="relu", nngp_prior=lambda: {"var_b": P.sample("var_b", pb), "var_w": P.sample("var_w", pw)})
    m2.X_train, m2.y_train = X, y
    plj = ProgramLogJoint(m2, lik=cpu_lik(m2, X))
    assert isinstance(make_log_joint(m2), ProgramLogJoint)
    assert [s.name for s in plj.sites] == ["var_b", "var_w", "noise"]
    for jac in (False, True):
        va, ga = lj(u, jac)
        vb, gb = plj(u, jac)
        assert abs(va - vb) < 1e-10 * abs(va)
        np.testing.assert_allclose(gb, ga, rtol=1e-6, atol=1e-7)
    np.testing.assert_array_equal(plj._run(u)[0], th)


def test_prior_draws_use_the_nngp_sites():
    from gpax_b200.inference import prior_draws
    m = vi_iBNN(2)
    draws = prior_draws(m, np.random.default_rng(0), 5, 2)
    assert len(draws) == 5 and all(set(kp) == {"var_b", "var_w"} and noise > 0 for kp, noise, _ in draws)


def test_acquisition_takes_finite_differences():
    m = iBNN(1)
    assert acquisition._analytic_kind(acquisition.EI, m, {}) is None
    assert acquisition._analytic_kind(acquisition.UCB, vi_iBNN(1), {}) is None
    m.X_train, m.y_train = _data()
    with pytest.raises(NotImplementedError):
        m._posterior_grad(np.zeros((2, 1)), {"var_b": 1.0, "var_w": 1.0, "noise": 0.1}, False, False)
