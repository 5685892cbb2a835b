"""CPU checks of deep kernel learning: the NumPy oracle's gradients against central differences, the haiku <-> flat
parameter layouts, DKL's site names, priors.Cauchy and the refused options."""
import numpy as np
import pytest
import scipy.stats as st

from gpax_b200 import DKL, viDKL
from gpax_b200 import priors as P
from oracle import dkl_oracle as dko
from oracle import fit_oracle as fo

KINDS = ["RBF", "Matern", "Periodic"]


def _problem(N=24, D=5, widths=(6, 4, 2), seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (N, D))
    X[3] = X[7]                                    # duplicate inputs
    y = np.sin(2 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    layers, i = [], D
    for w in widths:
        layers.append((rng.standard_normal((i, w)) / np.sqrt(i), 0.3 * rng.standard_normal(w)))
        i = w
    d = widths[-1]
    theta = np.r_[rng.uniform(0.5, 1.5, d), 1.3, 0.1, 1.7]
    return X, y, layers, theta


def _fd(f, x, h=1e-6):
    g = np.zeros_like(x)
    for k in range(x.size):
        e = np.zeros_like(x)
        e.flat[k] = h
        g.flat[k] = (f(x + e) - f(x - e)) / (2 * h)
    return g


@pytest.mark.parametrize("kind", KINDS)
def test_oracle_dz_matches_central_differences(kind):
    rng = np.random.default_rng(1)
    Z = rng.uniform(-1, 1, (20, 3))
    Z[4] = Z[11]                                   # duplicates: the derivative of the pair vanishes
    y = rng.standard_normal(20)
    theta = np.r_[0.7, 1.1, 0.9, 1.2, 0.05, 1.6]   # ARD lengthscales
    _, _, gz, _ = dko.mll_dz(kind, Z, y, theta, 1e-6)
    fd = _fd(lambda z: fo.mll_grad(kind, z.reshape(Z.shape), y, theta, 1e-6)[0], Z.copy())
    np.testing.assert_allclose(gz, fd, rtol=1e-6, atol=1e-6 * np.abs(fd).max())


@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("kind", ["RBF", "Matern"])
def test_oracle_weight_gradients_match_central_differences(kind, act):
    X, y, layers, theta = _problem()
    D, widths = X.shape[1], [w.shape[1] for w, _ in layers]
    flat = dko.flatten(layers)
    _, _, gp, _, _ = dko.dkl_mll(kind, X, y, layers, act, theta, 1e-6)
    fd = _fd(lambda p: dko.dkl_mll(kind, X, y, dko.unflatten(p, D, widths), act, theta, 1e-6)[0], flat.copy())
    np.testing.assert_allclose(gp, fd, rtol=1e-5, atol=1e-6 * np.abs(fd).max())


@pytest.mark.parametrize("kind", KINDS)
def test_oracle_log_theta_gradient(kind):
    X, y, layers, theta = _problem()
    _, g, _, _, _ = dko.dkl_mll(kind, X, y, layers, "tanh", theta, 1e-6)
    lt = np.log(theta)
    fd = _fd(lambda u: dko.dkl_mll(kind, X, y, layers, "tanh", np.exp(u), 1e-6)[0], lt.copy())
    if kind != "Periodic":
        fd[-1] = 0.0                               # period does not enter RBF / Matern
    np.testing.assert_allclose(g, fd, rtol=1e-6, atol=1e-7 * np.abs(fd).max())


def test_oracle_vidkl_loss_gradient():
    X, y, layers, theta = _problem()
    D, widths = X.shape[1], [w.shape[1] for w, _ in layers]
    v = np.concatenate([np.log(theta[:4]), dko.flatten(layers)])
    f = lambda p: dko.vidkl_loss("RBF", X, y, p[:4], p[4:], D, widths, "relu", 1e-6)   # noqa: E731
    _, g = f(v)
    fd = _fd(lambda p: f(p)[0], v.copy())
    np.testing.assert_allclose(g, fd, rtol=1e-5, atol=1e-6 * np.abs(fd).max())


def test_haiku_flat_round_trip():
    m = viDKL(7, z_dim=3)
    rng = np.random.default_rng(2)
    hk = {"mlp/~/linear": {"w": rng.standard_normal((7, 64)), "b": rng.standard_normal(64)},
          "mlp/~/linear_1": {"w": rng.standard_normal((64, 64)), "b": rng.standard_normal(64)},
          "mlp/~/linear_2": {"w": rng.standard_normal((64, 3)), "b": rng.standard_normal(3)}}
    flat = m.to_flat(hk)
    assert flat.shape == (7 * 64 + 64 + 64 * 64 + 64 + 64 * 3 + 3,)
    np.testing.assert_array_equal(flat[:7 * 64], hk["mlp/~/linear"]["w"].ravel())
    back = m.from_flat(flat)
    for k in hk:
        for p in ("w", "b"):
            np.testing.assert_array_equal(back[k][p], hk[k][p])
    stacked = {k: {p: np.stack([v[p], 2 * v[p]]) for p in v} for k, v in hk.items()}   # two channels
    fl2 = m.to_flat(stacked)
    assert fl2.shape == (2, flat.size)
    np.testing.assert_array_equal(fl2[1], 2 * flat)


@pytest.mark.parametrize("hidden", [None, [16, 8, 4]])
def test_dkl_site_names_and_shapes(hidden):
    m = DKL(10, z_dim=2, hidden_dim=hidden)
    h = [64, 32] if hidden is None else hidden
    assert m.site_names() == [n for i in range(len(h) + 1) for n in (f"w{i}", f"b{i}")]
    sizes = [10] + h + [2]
    flat = np.arange(sum(a * b + b for a, b in zip(sizes[:-1], sizes[1:])), dtype=float)
    d = m.from_flat(np.stack([flat, flat]))
    for i, (a, b) in enumerate(zip(sizes[:-1], sizes[1:])):
        assert d[f"w{i}"].shape == (2, a, b) and d[f"b{i}"].shape == (2, b)
    np.testing.assert_array_equal(m.to_flat(d)[0], flat)


def test_cauchy_prior_matches_scipy():
    c = P.Cauchy(0.3, 1.7)
    t = np.linspace(-10, 10, 41)
    np.testing.assert_allclose(c.log_prob(t), st.cauchy(0.3, 1.7).logpdf(t), rtol=1e-13)
    h = 1e-6
    np.testing.assert_allclose(c.dlog_prob(t), (c.log_prob(t + h) - c.log_prob(t - h)) / (2 * h), rtol=1e-7, atol=1e-9)
    np.testing.assert_array_equal(c.transform(t), t)
    np.testing.assert_array_equal(c.dtheta_du(t), np.ones_like(t))
    assert c.median() == 0.3 and float(c.log_abs_jac(1.0)) == 0.0


def test_refused_options():
    with pytest.raises(NotImplementedError):
        viDKL(5, nn=lambda x: x)
    with pytest.raises(NotImplementedError):
        viDKL(5, latent_prior=lambda z: z)
    with pytest.raises(NotImplementedError):
        viDKL((8, 8, 1))
    with pytest.raises(NotImplementedError):
        DKL(5, nn=lambda x, p: x)
    with pytest.raises(NotImplementedError):
        DKL(5, latent_prior=lambda z: z)
    with pytest.raises(NotImplementedError):
        DKL((4, 4))
    assert viDKL((6,)).data_dim == (6,)
