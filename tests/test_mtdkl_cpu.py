"""CPU: the NumPy oracle of multi-task deep kernel learning (oracle/mtdkl_oracle.py) against central differences, the
viMTDKL host layer (sites, shapes, the haiku <-> flat layout, the helpers shared with MultiTaskGP) and the refused
options."""
import numpy as np
import pytest

from oracle import dkl_oracle as dko
from oracle import mtdkl_oracle as mdo

JIT = 1e-6


def problem(n, D, widths, T, L, R, shared, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (n, D))
    task = np.tile(np.arange(T), n) if shared else rng.integers(0, T, n)
    y = rng.standard_normal(n * T if shared else n)
    layers, i = [], D
    for w in widths:
        layers.append((rng.standard_normal((i, w)) / np.sqrt(i), 0.2 * rng.standard_normal(w)))
        i = w
    d = widths[-1] if widths else D
    params = {"k_length": rng.uniform(0.5, 1.2, (L, d)), "k_scale": rng.uniform(0.8, 1.3, L), "W": rng.normal(0, 0.7, (L, T, R)),
              "v": np.exp(rng.normal(-1, 0.3, (L, T))), "noise": np.exp(rng.normal(-2.0, 0.3, T))}
    return X, task, y, layers, params


def fd(f, x, h):
    g = np.zeros(x.size)
    for k in range(x.size):
        e = np.zeros(x.size)
        e[k] = h
        e = e.reshape(x.shape)
        g[k] = (f(x + e) - f(x - e)) / (2 * h)
    return g.reshape(x.shape)


CASES = [(k, s, T, L) for k in ("RBF", "Matern") for s in (False, True) for T in (2, 3) for L in (1, 2)]


@pytest.mark.parametrize("kind,shared,T,L", CASES)
def test_dz_and_dparams_match_central_differences(kind, shared, T, L):
    widths = [5, 2]
    X, task, y, layers, params = problem(7 if shared else 14, 3, widths, T, L, 1, shared, seed=T * 10 + L)
    value, g_th, g_B, g_n, gp, gz, _ = mdo.mtdkl_mll(kind, X, task, y, layers, "tanh", params, shared, T, JIT)
    Z = dko.mlp_forward(X, layers, "tanh")[-1]
    fz = lambda z: mdo.lcm_dz(kind, z, task, y, params, shared, T, JIT)[0]    # noqa: E731
    np.testing.assert_allclose(gz, fd(fz, Z, 1e-5), rtol=1e-5, atol=1e-6 * np.abs(gz).max())
    flat = dko.flatten(layers)
    fp = lambda p: mdo.mtdkl_mll(kind, X, task, y, dko.unflatten(p, 3, widths), "tanh", params, shared, T, JIT)[0]  # noqa: E731
    np.testing.assert_allclose(gp, fd(fp, flat, 1e-5), rtol=1e-5, atol=1e-6 * np.abs(gp).max())
    # d / (log k_length, log k_scale), d / B_q (entries independent, symmetric part), d / log noise
    def with_(name, val):
        return mdo.mtdkl_mll(kind, X, task, y, layers, "tanh", dict(params, **{name: val}), shared, T, JIT)[0]
    g = fd(lambda u: with_("k_length", np.exp(u)), np.log(params["k_length"]), 1e-5)
    np.testing.assert_allclose(g_th[:, :2], g, rtol=1e-5, atol=1e-7)
    g = fd(lambda u: with_("k_scale", np.exp(u)), np.log(params["k_scale"]), 1e-5)
    np.testing.assert_allclose(g_th[:, 2], g, rtol=1e-5, atol=1e-7)
    g = fd(lambda u: with_("noise", np.exp(u)), np.log(params["noise"]), 1e-5)
    np.testing.assert_allclose(g_n, g, rtol=1e-5, atol=1e-7)
    g = fd(lambda v: with_("v", v), params["v"], 1e-6)
    np.testing.assert_allclose(np.diagonal(g_B, axis1=1, axis2=2), g, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("shared", [False, True])
def test_loss_gradient_matches_central_differences(shared):
    T, L, R, widths = 3, 2, 2, [4, 2]
    X, task, y, layers, params = problem(5 if shared else 12, 3, widths, T, L, R, shared, seed=3)
    u = np.concatenate([np.log(params["k_length"]).ravel(), 1.0 + 1e-5 * np.arange(L), params["W"].ravel(),
                        np.log(params["v"]).ravel(), np.log(params["noise"])])
    flat = dko.flatten(layers)
    v0 = np.concatenate([u, flat])
    nu = u.size
    f = lambda v: mdo.vimtdkl_loss("Matern", X, task, y, v[:nu], v[nu:], 3, widths, "relu", L, T, R, shared)   # noqa: E731
    loss, g = f(v0)
    ref = fd(lambda v: f(v)[0], v0, 1e-6)
    ref[L * 2:L * 3] = fd(lambda v: f(v)[0], v0, 1e-9)[L * 2:L * 3]     # k_scale: the Normal(1, 1e-4) prior is sharp
    np.testing.assert_allclose(g, ref, rtol=2e-5, atol=1e-5 * np.abs(g[nu:]).max())


# ---------------------------------------------------------------- the host layer
def test_sites_shapes_and_layout():
    from gpax_b200 import viMTDKL
    m = viMTDKL(4, z_dim=3, num_latents=2, rank=1)
    X = np.column_stack([np.zeros((9, 4)), np.arange(9) % 3])
    m.X_train = X
    sites = [(n, sh) for n, _, sh in m._site_list()]
    assert sites == [("k_length", (2, 3)), ("k_scale", (2, 1)), ("W", (2, 3, 1)), ("v", (2, 3)), ("noise", (3,))]
    m2 = viMTDKL(4, num_tasks=2, shared_input_space=True)       # L = T, rank = T - 1
    m2.X_train = np.zeros((5, 4))
    assert [sh for _, _, sh in m2._site_list()] == [(2, 2), (2, 1), (2, 2, 1), (2, 2), (2,)]
    rng = np.random.default_rng(0)
    flat = rng.standard_normal(4 * 64 + 64 + 64 * 64 + 64 + 64 * 3 + 3)
    nn = m.from_flat(flat)
    assert list(nn) == ["mlp/~/linear", "mlp/~/linear_1", "mlp/~/linear_2"] and nn["mlp/~/linear_2"]["w"].shape == (64, 3)
    assert np.array_equal(m.to_flat(nn), flat)


def test_w_starts_off_its_stationary_median():
    from gpax_b200 import viMTDKL
    m = viMTDKL(4, num_latents=2)
    m.X_train = np.column_stack([np.zeros((6, 4)), np.arange(6) % 3])
    u, flat = m._init_params(np.random.default_rng(1))
    kp = m._theta(u)
    assert np.all(kp["W"] != 0) and np.allclose(kp["k_length"], 1) and np.allclose(kp["k_scale"], 1)
    assert np.allclose(kp["v"], 1) and np.allclose(kp["noise"], 1) and flat.size == 4 * 64 + 64 + 64 * 64 + 64 + 64 * 2 + 2


def test_points_and_task_matrix_helpers_keep_multitaskgp_behaviour():
    from gpax_b200 import MultiTaskGP
    from gpax_b200.mtgp import lcm_points, lcm_task_matrix
    rng = np.random.default_rng(2)
    W, v = rng.standard_normal((2, 3, 3, 2)), rng.uniform(0.1, 1, (2, 3, 3))
    B = np.einsum("sltr,slur->sltu", W, W) + v[..., None] * np.eye(3)
    np.testing.assert_allclose(lcm_task_matrix(W, v), B, rtol=1e-15)
    X = np.column_stack([rng.standard_normal((5, 2)), [0, 2, 1, 1, 0]])
    m = MultiTaskGP(2, "RBF", num_latents=1, num_tasks=3)
    rows, t, g = m._rows(X)
    assert g == 1 and np.array_equal(rows, X[:, :2]) and list(t) == [0, 2, 1, 1, 0]
    with pytest.raises(ValueError):
        lcm_points(np.column_stack([X[:, :2], [0, 3, 1, 1, 0]]), 3, False)
    k = MultiTaskGP(2, "RBF", shared_input_space=True, num_tasks=3)
    rows, t, g = k._rows(X[:, :2])
    assert g == 3 and np.array_equal(rows, np.repeat(X[:, :2], 3, 0)) and list(t) == [0, 1, 2] * 5


def test_refused_options():
    from gpax_b200 import viMTDKL
    with pytest.raises(NotImplementedError):
        viMTDKL(3, data_kernel="Periodic", num_latents=1)
    with pytest.raises(NotImplementedError):
        viMTDKL(3, num_latents=1, data_kernel_prior=lambda: {})
    with pytest.raises(NotImplementedError):
        viMTDKL(3, num_latents=1, task_kernel_prior=lambda: {})
    with pytest.raises(NotImplementedError):
        viMTDKL(3, num_latents=1, nn=lambda x: x)
    with pytest.raises(ValueError):
        viMTDKL(3)                                            # multitask form needs num_latents
    with pytest.raises(ValueError):
        viMTDKL(3, shared_input_space=True)                   # Kronecker form needs num_tasks
