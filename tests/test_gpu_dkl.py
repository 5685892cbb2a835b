"""Deep kernel learning on the GPU: b2gp_dkl_mll and b2gp_mlp_forward against the NumPy oracle (oracle/dkl_oracle.py) on
the fp64 and int8 solve routes, bit-identity with b2gp_mll, the failure path, and the viDKL / DKL models end to end."""
import numpy as np
import pytest

from oracle import dkl_oracle as dko

pytestmark = pytest.mark.gpu

ACT = {"relu": 0, "tanh": 1}
JIT = 1e-6


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def _problem(N, D, widths, seed, kind="RBF"):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (N, D))
    y = np.sin(3 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    layers, i = [], D
    for w in widths:
        layers.append((rng.standard_normal((i, w)) / np.sqrt(i), 0.2 * rng.standard_normal(w)))
        i = w
    d = widths[-1] if widths else D
    theta = np.r_[rng.uniform(0.6, 1.2, d), 1.2, 0.1, 1.5]
    return X, y, layers, theta


def _close(got, ref, tol, what):
    scale = max(np.abs(ref).max(), 1e-300)
    err = np.abs(np.asarray(got) - ref).max()
    assert err <= tol * scale, f"{what}: max error {err:.3e} vs scale {scale:.3e}"


CASES = [(k, a, L, N) for k in ("RBF", "Matern", "Periodic") for a in ("relu", "tanh") for L in (0, 3) for N in (300, 2500)]


@pytest.mark.parametrize("ozaki", [0, 7])
@pytest.mark.parametrize("kind,act,L,N", CASES)
def test_dkl_mll_matches_oracle(ctx, kind, act, L, N, ozaki):
    D = 12 if L else 2
    widths = [16, 8, 2][:L]
    X, y, layers, theta = _problem(N, D, widths, seed=N + L, kind=kind)
    with ctx.options(ozaki=ozaki):
        val, g, gp, gz, info = ctx.dkl_mll(kind, X, y, widths, ACT[act], dko.flatten(layers) if L else np.zeros(0), theta, JIT,
                                           want_params=True, want_z=True)
    assert info == 0
    rv, rg, rgp, rgz, _ = dko.dkl_mll(kind, X, y, layers, act, theta, JIT)
    assert abs(val - rv) <= 1e-9 * max(1.0, abs(rv))
    _close(g, rg, 1e-8, "grad_theta")
    _close(gz, rgz, 1e-8, "grad_z")
    if L:
        _close(gp, rgp, 1e-8, "grad_params")


@pytest.mark.parametrize("N", [300, 2500, 9000])
def test_value_and_grad_theta_bit_identical_to_mll(ctx, N):
    """the value and grad_theta are b2gp_mll's on the same z (9000: the fp64 tall-panel route)"""
    widths = [16, 8, 2]
    X, y, layers, theta = _problem(N, 12, widths, seed=7)
    flat = dko.flatten(layers)
    with ctx.options(ozaki=0):
        val, g, gp, gz, info = ctx.dkl_mll("Matern", X, y, widths, ACT["relu"], flat, theta, JIT, want_z=True)
        Z = ctx.mlp_forward(X, widths, ACT["relu"], flat)[0]
        mv, mg, _, minfo = ctx.mll("Matern", Z, y, theta, JIT)
    assert info == minfo == 0
    assert val == mv and np.array_equal(g, mg)
    assert np.isfinite(gp).all() and np.isfinite(gz).all()
    val2, g2, gp2, gz2, _ = ctx.dkl_mll("Matern", X, y, widths, ACT["relu"], flat, theta, JIT, want_z=True)
    assert val2 == val and np.array_equal(gp2, gp) and np.array_equal(gz2, gz)     # deterministic


def test_device_and_host_pointers_agree(ctx):
    widths = [16, 8, 2]
    X, y, layers, theta = _problem(500, 12, widths, seed=3)
    flat = dko.flatten(layers)
    host = ctx.dkl_mll("RBF", X, y, widths, ACT["tanh"], flat, theta, JIT, want_z=True)
    Xd, yd = ctx.to_device(X), ctx.to_device(y)
    try:
        dev = ctx.dkl_mll("RBF", Xd, yd, widths, ACT["tanh"], flat, theta, JIT, want_z=True)
    finally:
        Xd.free()
        yd.free()
    assert host[0] == dev[0] and host[4] == dev[4]
    for a, b in zip(host[1:4], dev[1:4]):
        assert np.array_equal(a, b)


def test_indefinite_kernel_gives_nan(ctx):
    widths = [16, 8, 2]
    X, y, layers, theta = _problem(200, 12, widths, seed=4)
    theta[3] = -5.0                                 # negative noise: K is indefinite
    val, g, gp, gz, info = ctx.dkl_mll("RBF", X, y, widths, ACT["relu"], dko.flatten(layers), theta, JIT, want_z=True)
    assert info != 0
    assert np.isnan(val) and np.isnan(g).all() and np.isnan(gp).all() and np.isnan(gz).all()


@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_mlp_forward_weight_sets(ctx, act):
    widths = [64, 32, 3]
    rng = np.random.default_rng(5)
    X = rng.standard_normal((777, 40))
    sets = [_problem(2, 40, widths, seed=s)[2] for s in range(4)]
    Z = ctx.mlp_forward(X, widths, ACT[act], np.stack([dko.flatten(ls) for ls in sets]))
    assert Z.shape == (4, 777, 3)
    for s, ls in enumerate(sets):
        ref = dko.mlp_forward(X, ls, act)[-1]
        _close(Z[s], ref, 1e-12, f"set {s}")


def test_vidkl_posterior_and_predict_match_oracle():
    from gpax_b200 import viDKL
    rng = np.random.default_rng(6)
    X, Xn = rng.uniform(-1, 1, (40, 12)), rng.uniform(-1, 1, (15, 12))
    y = np.cos(2 * X[:, 1]) + 0.05 * rng.standard_normal(40)
    m = viDKL(12, z_dim=2, kernel="Matern")
    _, _, layers, _ = _problem(2, 12, [64, 64, 2], seed=8)
    nn = m.from_flat(dko.flatten(layers))
    kp = {"k_length": np.array([0.8, 1.1]), "k_scale": np.array(1.3), "noise": np.array(0.02)}
    m.X_train, m.y_train = X, y
    for noiseless in (False, True):
        mean, cov = m.get_mvn_posterior(Xn, nn, kp, noiseless)
        rm, rc = dko.posterior("Matern", X, y, Xn, layers, "relu", kp, noiseless)
        _close(mean, rm, 1e-9, "mean")
        _close(cov, rc, 1e-9, "cov")
    m.nn_params, m.kernel_params = nn, kp
    mean, var = m.predict(0, Xn)
    rm, rc = dko.posterior("Matern", X, y, Xn, layers, "relu", kp)
    _close(mean, rm, 1e-9, "predict mean")
    _close(var, np.diag(rc), 1e-9, "predict var")
    # three channels: stacked leaves, one embedding per channel
    Y = np.stack([y, 2 * y, y ** 2])
    sets = [_problem(2, 12, [64, 64, 2], seed=20 + c)[2] for c in range(3)]
    m.y_train = Y
    m.nn_params = m.from_flat(np.stack([dko.flatten(s) for s in sets]))
    m.kernel_params = {k: np.stack([np.asarray(v) * (1 + 0.1 * c) for c in range(3)]) for k, v in kp.items()}
    mean, var = m.predict(0, Xn)
    assert mean.shape == var.shape == (3, 15)
    for c in range(3):
        kc = {k: v[c] for k, v in m.kernel_params.items()}
        rm, rc = dko.posterior("Matern", X, Y[c], Xn, sets[c], "relu", kc)
        _close(mean[c], rm, 1e-9, f"channel {c} mean")
        _close(var[c], np.diag(rc), 1e-9, f"channel {c} var")
    assert m.embed(Xn).shape == (3, 15, 2)


def test_vidkl_adam_matches_oracle():
    """25 Adam steps of viDKL.fit from one fixed initialisation against the oracle's Adam on the same loss"""
    from gpax_b200 import viDKL
    rng = np.random.default_rng(9)
    X = rng.uniform(-1, 1, (60, 6))
    y = np.sin(2 * X[:, 0] + X[:, 1]) + 0.05 * rng.standard_normal(60)
    m = viDKL(6, z_dim=2, kernel="RBF")
    _, _, layers, _ = _problem(2, 6, [64, 64, 2], seed=10)
    flat0 = dko.flatten(layers)
    m._init_params = lambda r: (np.zeros(4), flat0.copy())
    m.fit(0, X, y, num_steps=25, step_size=5e-3, print_summary=False, progress_bar=False)
    f = lambda p: dko.vidkl_loss("RBF", X, y, p[:4], p[4:], 6, [64, 64, 2], "relu", JIT)   # noqa: E731
    ref, _ = dko.adam(f, np.concatenate([np.zeros(4), flat0]), 25, 5e-3)
    np.testing.assert_allclose(m.loss, ref, rtol=1e-7)


def test_fit_predict_ensemble_shapes():
    from gpax_b200 import viDKL
    rng = np.random.default_rng(12)
    X, Xn = rng.uniform(-1, 1, (30, 5)), rng.uniform(-1, 1, (7, 5))
    y = X[:, 0] ** 2
    m = viDKL(5)
    mean, var = m.fit_predict(0, X, y, Xn, num_steps=5, n_models=3, print_summary=False, progress_bar=False)
    assert mean.shape == var.shape == (3, 7) and np.isfinite(mean).all()
    mean, var = m.fit_predict(0, X, np.stack([y, -y]), Xn, num_steps=5, n_models=3, print_summary=False, progress_bar=False)
    assert mean.shape == var.shape == (3, 2, 7) and np.isfinite(var).all()


def test_dkl_nuts_sites_and_predict():
    from gpax_b200 import DKL
    rng = np.random.default_rng(13)
    X, Xn = rng.uniform(-1, 1, (100, 8)), rng.uniform(-1, 1, (9, 8))
    y = np.sin(2 * X[:, 0]) + 0.05 * rng.standard_normal(100)
    m = DKL(8, z_dim=2, hidden_dim=[8, 4])
    m.fit(0, X, y, num_warmup=10, num_samples=6, progress_bar=False, print_summary=False)
    s = m.get_samples()
    shapes = {"w0": (8, 8), "b0": (8,), "w1": (8, 4), "b1": (4,), "w2": (4, 2), "b2": (2,), "k_length": (2,), "k_scale": (),
              "noise": ()}
    assert set(s) == set(shapes)
    for k, sh in shapes.items():
        assert s[k].shape == (6,) + sh, k
    mean, ys = m.predict(0, Xn, n=2)
    assert ys.shape == (6, 2, 9)
    means = []
    for i in range(6):
        p = {k: v[i] for k, v in s.items()}
        layers = [(p[f"w{l}"], p[f"b{l}"]) for l in range(3)]
        rm, _ = dko.posterior("RBF", X, y, Xn, layers, "tanh", p)
        means.append(rm)
        gm, _ = m.get_mvn_posterior(Xn, p)
        _close(gm, rm, 1e-9, f"draw {i} mean")
    _close(mean, np.mean(means, 0), 1e-9, "mean over draws")
    assert m.embed(Xn).shape == (6, 9, 2)


# ---------------------------------------------------------------- against the reference's own vidkl.py / dkl.py
def _golden():
    import os
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_dkl.npz"))


HK = ["mlp/~/linear", "mlp/~/linear_1", "mlp/~/linear_2"]


def test_vidkl_matches_golden():
    from gpax_b200 import viDKL
    G = _golden()
    m = viDKL(12, z_dim=2, kernel="RBF")
    m.X_train, m.y_train = G["X"], G["y"]
    nn = {n: {"w": G[f"vidkl_{n}_w"], "b": G[f"vidkl_{n}_b"]} for n in HK}
    kp = {"k_length": np.array([0.8, 1.1]), "k_scale": np.array(1.3), "noise": np.array(0.02)}
    for nl in (False, True):
        mean, cov = m.get_mvn_posterior(G["X_new"], nn, kp, nl)
        _close(mean, G[f"vidkl_mean_noiseless{int(nl)}"], 1e-9, "mean")
        _close(cov, G[f"vidkl_cov_noiseless{int(nl)}"], 1e-9, "cov")
    m.nn_params, m.kernel_params = nn, kp
    mean, var = m.predict(0, G["X_new"])
    _close(mean, G["vidkl_predict_mean"], 1e-9, "predict mean")
    _close(var, G["vidkl_predict_var"], 1e-9, "predict var")
    _close(m.embed(G["X_new"]), G["vidkl_embed"], 1e-12, "embed")
    m.y_train = G["vidkl3_Y"]
    m.nn_params = {n: {"w": G[f"vidkl3_{n}_w"], "b": G[f"vidkl3_{n}_b"]} for n in HK}
    m.kernel_params = {k: G[f"vidkl3_{k}"] for k in ("k_length", "k_scale", "noise")}
    mean, var = m.predict(0, G["X_new"])
    _close(mean, G["vidkl3_predict_mean"], 1e-9, "3-channel mean")
    _close(var, G["vidkl3_predict_var"], 1e-9, "3-channel var")


@pytest.mark.parametrize("tag,hidden", [("default", None), ("custom", [16, 8, 4])])
def test_dkl_matches_golden(tag, hidden):
    from gpax_b200 import DKL
    from gpax_b200.inference import MCMCResult
    G = _golden()
    m = DKL(12, z_dim=2, kernel="Matern", hidden_dim=hidden)
    m.X_train, m.y_train = G["X"], G["y"]
    params = {k[len(f"dkl_{tag}_"):]: G[k] for k in G.files if k.startswith(f"dkl_{tag}_") and
              not k.endswith(("_mean", "_cov", "_embed"))}
    mean, cov = m.get_mvn_posterior(G["X_new"], params)
    _close(mean, G[f"dkl_{tag}_mean"], 1e-9, "mean")
    _close(cov, G[f"dkl_{tag}_cov"], 1e-9, "cov")
    m.mcmc = MCMCResult({k: np.stack([np.stack([v, 1.1 * v])]) for k, v in params.items()}, [{}])
    _close(m.embed(G["X_new"]), G[f"dkl_{tag}_embed"], 1e-12, "embed")


# ---------------------------------------------------------------- acquisition functions on the embeddings
def test_acquisitions_on_dkl_use_the_embedding():
    from gpax_b200 import DKL, acquisition
    from gpax_b200.inference import MCMCResult
    rng = np.random.default_rng(14)
    X, Xn = rng.uniform(-1, 1, (50, 6)), rng.uniform(-1, 1, (11, 6))
    y = np.sin(2 * X[:, 0]) + 0.05 * rng.standard_normal(50)
    m = DKL(6, z_dim=2, hidden_dim=[8, 4])
    m.X_train, m.y_train = X, y
    S = 4
    draws = [_problem(2, 6, [8, 4, 2], seed=30 + s)[2] for s in range(S)]
    samples = {}
    for l in range(3):
        samples[f"w{l}"] = np.stack([d[l][0] for d in draws])
        samples[f"b{l}"] = np.stack([d[l][1] for d in draws])
    samples.update({"k_length": rng.uniform(0.6, 1.2, (S, 2)), "k_scale": np.full(S, 1.1), "noise": np.full(S, 0.05)})
    m.mcmc = MCMCResult({k: v[None] for k, v in samples.items()}, [{}])
    out = m._posterior_batched(Xn, samples, True, False, ("mean", "var"))
    for s in range(S):
        p = {k: v[s] for k, v in samples.items()}
        rm, rc = dko.posterior("RBF", X, y, Xn, draws[s], "tanh", p)
        _close(out["mean"][s], rm, 1e-9, f"draw {s} mean")
        _close(out["var"][s], np.diag(rc), 1e-9, f"draw {s} var")
    q = acquisition.qEI(0, m, Xn, subsample_size=2, n_evals=3)
    assert np.isfinite(np.asarray(q, dtype=float)).all()
    kg = acquisition.KG(0, m, Xn, n=3)
    assert np.asarray(kg).shape == (S, 11) and np.isfinite(kg).all()


def test_vidkl_options_and_batches():
    """nn_prior=False with the normal guide (weights stay point parameters), Periodic, and predict_in_batches' merged
    chunks agreeing with one predict call; KG on the fitted model"""
    from gpax_b200 import viDKL, acquisition
    rng = np.random.default_rng(15)
    X, Xn = rng.uniform(-1, 1, (60, 5)), rng.uniform(-1, 1, (9000, 5))
    y = np.sin(2 * X[:, 0]) + 0.05 * rng.standard_normal(60)
    m = viDKL(5, z_dim=2, kernel="Periodic", nn_prior=False, guide="normal")
    m.fit(0, X, y, num_steps=20, print_summary=False, progress_bar=False)
    assert np.isfinite(m.loss).all() and set(m.kernel_params) == {"k_length", "k_scale", "noise", "period"}
    mean, var = m.predict(0, Xn)
    mb, vb = m.predict_in_batches(0, Xn, batch_size=100)
    _close(mb, mean, 1e-12, "batched mean")
    _close(vb, var, 1e-12, "batched var")
    kg = acquisition.KG(0, m, Xn[:7], n=3)
    assert np.asarray(kg).shape == (7,) and np.isfinite(kg).all()
