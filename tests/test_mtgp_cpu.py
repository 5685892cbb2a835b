"""CPU: the multi-task oracle, the host model programs, parameter packing and the refusals of MultiTaskGP / CoregGP."""
import numpy as np
import pytest

from oracle import mtgp_oracle as mo


def rand_params(rng, L, T, R, d, kind):
    return {"k_length": rng.uniform(0.5, 1.5, (L, d)), "k_scale": rng.uniform(0.5, 1.5, L), "W": rng.normal(size=(L, T, R)),
            "v": rng.uniform(0.5, 1.0, (L, T)), "noise": rng.uniform(0.1, 0.3, T),
            "period": rng.uniform(1.0, 2.0, L) if kind == "Periodic" else None}


def test_lcm_cov_matches_the_reference_lcm_kernel(gf):
    prm = {k: gf["lcm_" + k] for k in ("k_length", "k_scale", "W", "v")}
    nt = np.array([0.01, 0.02, 0.03])
    np.testing.assert_allclose(mo.lcm_cov(gf["mt_X"], gf["mt_X"], prm, nt, "RBF"), gf["lcm_XX"], rtol=1e-13)


def test_lcm_cov_adds_noise_once_per_latent_and_jitter_times_B():
    """consequences 1 and 2: diagonal sum_q (k_q(x,x) + jitter) B_q[t,t] + L (noise[t] + jitter); Kronecker jitter on the block"""
    rng = np.random.default_rng(1)
    L, T, d = 2, 3, 2
    p = rand_params(rng, L, T, 2, d, "Matern")
    X = rng.uniform(0, 1, (4, d))
    K = mo.lcm_cov(X, X, p, p["noise"], "Matern", True, T, jitter=1e-3)
    B = np.einsum("qtr,qsr->qts", p["W"], p["W"]) + np.stack([np.diag(v) for v in p["v"]])
    kxx = p["k_scale"] * (1 + np.sqrt(5) * 1e-6) * np.exp(-np.sqrt(5) * 1e-6)        # Matern k(x, x), consequence 5
    blk = sum((kxx[q] + 1e-3) * B[q] for q in range(L)) + L * np.diag(p["noise"] + 1e-3)
    np.testing.assert_allclose(K[:T, :T], blk, rtol=1e-13)


@pytest.mark.parametrize("kind,shared", [("RBF", False), ("Matern", True), ("Periodic", False)])
def test_oracle_gradient_matches_central_differences(kind, shared):
    rng = np.random.default_rng(2)
    L, T, R, d, n = 2, 3, 2, 2, 7
    if shared:
        X, y = rng.uniform(0, 1, (n, d)), rng.normal(size=n * T)
    else:
        X, y = np.c_[rng.uniform(0, 1, (2 * n, d)), rng.integers(0, T, 2 * n)], rng.normal(size=2 * n)
    p = rand_params(rng, L, T, R, d, kind)
    v, gt, gB, gn = mo.loglik_grad(X, y, p, kind, shared, T)
    assert abs(v - mo.loglik(X, y, p, kind, shared, T)) < 1e-12 * abs(v)
    h = 1e-6

    def fd(name, idx, logscale):
        pp = {k: (None if a is None else np.array(a, dtype=float)) for k, a in p.items()}
        pm = {k: (None if a is None else np.array(a, dtype=float)) for k, a in p.items()}
        if logscale:
            pp[name][idx] *= np.exp(h)
            pm[name][idx] *= np.exp(-h)
        else:
            pp[name][idx] += h
            pm[name][idx] -= h
        return (mo.loglik(X, y, pp, kind, shared, T) - mo.loglik(X, y, pm, kind, shared, T)) / (2 * h)

    for q in range(L):
        for k in range(d):
            assert abs(gt[q, k] - fd("k_length", (q, k), True)) < 1e-6
        assert abs(gt[q, d] - fd("k_scale", q, True)) < 1e-6
        if kind == "Periodic":
            assert abs(gt[q, d + 1] - fd("period", q, True)) < 1e-6
        gW = (gB[q] + gB[q].T) @ p["W"][q]
        for t in range(T):
            assert abs(gW[t, 1] - fd("W", (q, t, 1), False)) < 1e-6
            assert abs(gB[q, t, t] - fd("v", (q, t), False)) < 1e-6
    for t in range(T):
        assert abs(gn[t] - fd("noise", t, True)) < 1e-6


def test_existing_plates_keep_their_shapes():
    from gpax_b200 import priors as P

    def prog():
        with P.plate("a", 3):
            with P.plate("b", 2):
                x = P.sample("x", P.LogNormal(0.0, 1.0))
        return x
    _, sites, _ = P.run_program(prog)
    assert sites["x"].shape == (3, 2)


def test_packing_round_trips():
    from gpax_b200 import MultiTaskGP
    rng = np.random.default_rng(3)
    L, T, R, d, S = 2, 3, 2, 2, 4
    m = MultiTaskGP(d, "Periodic", num_latents=L, num_tasks=T)
    p = {"k_length": rng.uniform(size=(S, L, d)), "k_scale": np.ones((S, L)), "period": rng.uniform(size=(S, L, 1)),
         "W": rng.normal(size=(S, L, T, R)), "v": rng.uniform(size=(S, L, T)), "noise": rng.uniform(size=(S, T))}
    th, B, nz = m._pack(p, batched=True)
    assert th.shape == (S, L, d + 2) and B.shape == (S, L, T, T) and nz.shape == (S, T)
    np.testing.assert_array_equal(th[..., :d], p["k_length"])
    np.testing.assert_array_equal(th[..., d + 1], p["period"][..., 0])
    np.testing.assert_allclose(B[2, 1], p["W"][2, 1] @ p["W"][2, 1].T + np.diag(p["v"][2, 1]), rtol=1e-15)
    np.testing.assert_array_equal(nz, p["noise"])
    one = m._pack({k: v[1] for k, v in p.items()}, batched=False)
    for a, b in zip(one, (th[1:2], B[1:2], nz[1:2])):
        np.testing.assert_array_equal(a, b)


def test_task_labels_are_validated():
    from gpax_b200 import CoregGP, MultiTaskGP
    m = MultiTaskGP(1, "RBF", num_latents=1, num_tasks=2)
    m.X_train = np.c_[np.linspace(0, 1, 4), [0, 1, 0, 1]]
    Xd, t, g = m._rows(np.c_[np.linspace(0, 1, 3), [0, 1.9, 1]])
    assert t.tolist() == [0, 1, 1] and g == 1 and Xd.shape == (3, 1)
    with pytest.raises(ValueError):
        m._rows(np.c_[np.linspace(0, 1, 3), [0, 2, 1]])
    with pytest.raises(ValueError):
        m._rows(np.c_[np.linspace(0, 1, 3), [0, -1, 1]])
    k = MultiTaskGP(1, "RBF", shared_input_space=True, num_tasks=3)
    Xd, t, g = k._rows(np.linspace(0, 1, 2))
    assert Xd[:, 0].tolist() == [0, 0, 0, 1, 1, 1] and t.tolist() == [0, 1, 2, 0, 1, 2] and g == 3
    c = CoregGP(1, "RBF")
    c.X_train = np.c_[np.linspace(0, 1, 4), [0, 1, 2, 2]]
    assert c._num_tasks() == 3 and c._rank() == 1


def test_constructor_errors_and_refused_kernels():
    from gpax_b200 import CoregGP, MultiTaskGP
    with pytest.raises(ValueError, match="num_tasks"):
        MultiTaskGP(1, "RBF", shared_input_space=True)
    with pytest.raises(ValueError, match="num_latents"):
        MultiTaskGP(1, "RBF", shared_input_space=False)
    m = MultiTaskGP(1, "RBF", shared_input_space=True, num_tasks=3)
    assert m.num_latents == 3 and m.rank is None
    for bad in ("NNGP", lambda X, Z, p: X):
        with pytest.raises(NotImplementedError):
            MultiTaskGP(1, bad, num_latents=1)
        with pytest.raises(NotImplementedError):
            CoregGP(1, bad)


def test_oracle_posterior_is_the_explicit_inverse():
    """k_pX carries no diagonal term even when P = N (consequence 3); noiseless drops only the noise (consequence 4)"""
    rng = np.random.default_rng(4)
    L, T, d = 2, 2, 1
    p = rand_params(rng, L, T, 1, d, "RBF")
    X = np.c_[rng.uniform(0, 1, (6, d)), [0, 1, 0, 1, 0, 1]]
    y = rng.normal(size=6)
    m1, c1 = mo.posterior(X, y, X, p, "RBF")
    m0, c0 = mo.posterior(X, y, X, p, "RBF", noiseless=True)
    np.testing.assert_allclose(c1 - c0, np.diag(L * p["noise"][X[:, -1].astype(int)]), atol=1e-12)
    kpx = mo.lcm_cov(X, X, p, np.zeros(T), "RBF", jitter=0.0)
    np.testing.assert_allclose(m1, kpx @ np.linalg.solve(mo.lcm_cov(X, X, p, p["noise"], "RBF"), y), rtol=1e-9)


@pytest.fixture(scope="module")
def gf():
    import os
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_f.npz"))
