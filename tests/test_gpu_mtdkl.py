"""Multi-task deep kernel learning on the GPU: b2gp_mtdkl_mll against the NumPy oracle (oracle/mtdkl_oracle.py) on the
recursive, tall int8 and tall fp64 solve routes, bit-identity with b2gp_mll_multitask, the failure path, and viMTDKL end
to end (posterior, predict, the Adam loop, the reference's own test cases, acquisition functions)."""
import numpy as np
import pytest

from oracle import dkl_oracle as dko
from oracle import mtdkl_oracle as mdo

pytestmark = pytest.mark.gpu

ACT = {"relu": 0, "tanh": 1}
JIT = 1e-6


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def _problem(n, D, widths, T, L, R, shared, seed):
    """n points (n * T GP rows in the Kronecker form)"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (n, D))
    task = np.tile(np.arange(T), n) if shared else rng.integers(0, T, n)
    rows = n * T if shared else n
    y = np.sin(3 * np.repeat(X[:, 0], T if shared else 1)) + 0.3 * task + 0.1 * rng.standard_normal(rows)
    layers, i = [], D
    for w in widths:
        layers.append((rng.standard_normal((i, w)) / np.sqrt(i), 0.2 * rng.standard_normal(w)))
        i = w
    d = widths[-1] if widths else D
    params = {"k_length": rng.uniform(0.6, 1.2, (L, d)), "k_scale": rng.uniform(0.8, 1.3, L), "W": rng.normal(0, 0.7, (L, T, R)),
              "v": np.exp(rng.normal(-1, 0.3, (L, T))), "noise": np.exp(rng.normal(-2.0, 0.3, T))}
    return X, task, y, layers, params


def _abi(params):
    from gpax_b200.mtgp import lcm_task_matrix
    L, d = params["k_length"].shape
    theta = np.ones((L, d + 2))
    theta[:, :d], theta[:, d] = params["k_length"], params["k_scale"]
    return theta, lcm_task_matrix(params["W"], params["v"]), params["noise"]


def _close(got, ref, tol, what):
    scale = max(np.abs(ref).max(), 1e-300)
    err = np.abs(np.asarray(got) - ref).max()
    assert err <= tol * scale, f"{what}: max error {err:.3e} vs scale {scale:.3e}"


def _check(ctx, kind, shared, T, L, nl, n, ozaki, seed, act="relu"):
    D = 10 if nl else 2
    widths = [16, 8, 2][:nl]
    X, task, y, layers, params = _problem(n, D, widths, T, L, 2, shared, seed)
    theta, B, noise = _abi(params)
    group = T if shared else 1
    with ctx.options(ozaki=ozaki):
        val, gt, gB, gn, gp, gz, info = ctx.mtdkl_mll(kind, X, task, y, widths, ACT[act], dko.flatten(layers) if nl else np.zeros(0),
                                                      theta, B, noise, group, JIT, want_params=True, want_z=True)
    assert info == 0
    rv, rth, rB, rn, rgp, rgz, _ = mdo.mtdkl_mll(kind, X, task, y, layers, act, params, shared, T, JIT)
    assert abs(val - rv) <= 1e-9 * max(1.0, abs(rv))
    _close(gt, rth, 1e-8, "grad_theta")
    _close(gB, rB, 1e-8, "grad_B")
    _close(gn, rn, 1e-8, "grad_noise")
    _close(gz, rgz, 1e-8, "grad_z")
    if nl:
        _close(gp, rgp, 1e-8, "grad_params")


CASES = [(k, s, T, L, nl) for k in ("RBF", "Matern") for s in (False, True) for T in (2, 3) for L in (1, 2) for nl in (0, 3)]


@pytest.mark.parametrize("ozaki", [0, 7])
@pytest.mark.parametrize("kind,shared,T,L,nl", CASES)
def test_mtdkl_mll_matches_oracle(ctx, kind, shared, T, L, nl, ozaki):
    """about 300 GP rows: the recursive route"""
    _check(ctx, kind, shared, T, L, nl, 100 if shared else 300, ozaki, seed=T * 100 + L * 10 + nl)


@pytest.mark.parametrize("ozaki", [0, 7])
@pytest.mark.parametrize("kind,shared", [("RBF", False), ("Matern", True)])
def test_mtdkl_mll_matches_oracle_tall(ctx, kind, shared, ozaki):
    """about 2500 GP rows: the tall int8 route under ozaki = 7"""
    _check(ctx, kind, shared, 3, 2, 3, 834 if shared else 2500, ozaki, seed=5, act="tanh")


@pytest.mark.parametrize("shared,n", [(False, 300), (True, 834), (True, 3000)])
def test_value_and_grads_bit_identical_to_mll_multitask(ctx, shared, n):
    """value, grad_theta, grad_B and grad_noise are b2gp_mll_multitask's on the expanded z (3000 x 3 rows: the fp64 tall
    route); identical calls give identical bits"""
    T, L, widths = 3, 2, [16, 8, 2]
    X, task, y, layers, params = _problem(n, 10, widths, T, L, 2, shared, seed=7)
    theta, B, noise = _abi(params)
    flat, group = dko.flatten(layers), T if shared else 1
    with ctx.options(ozaki=0):
        out = ctx.mtdkl_mll("Matern", X, task, y, widths, ACT["relu"], flat, theta, B, noise, group, JIT, want_z=True)
        Z = ctx.mlp_forward(X, widths, ACT["relu"], flat)[0]
        mv, mg, mB, mn, _, minfo = ctx.mll_multitask("Matern", np.repeat(Z, group, axis=0), task, y, theta, B, noise, group, JIT)
        again = ctx.mtdkl_mll("Matern", X, task, y, widths, ACT["relu"], flat, theta, B, noise, group, JIT, want_z=True)
    val, gt, gB, gn, gp, gz, info = out
    assert info == minfo == 0
    assert val == mv and np.array_equal(gt, mg) and np.array_equal(gB, mB) and np.array_equal(gn, mn)
    assert np.isfinite(gp).all() and np.isfinite(gz).all()
    assert again[0] == val and all(np.array_equal(a, b) for a, b in zip(again[1:6], out[1:6]))
    if n >= 3000:
        # the fp64 tall route: d value / dz of a few points against a dense NumPy reference on the same z
        pts = [0, 1, n // 2, n - 1]
        ref, scale = _dense_dz_points("Matern", Z, y, params, T, pts)
        err = np.abs(gz[pts] - ref).max()
        assert err <= 1e-8 * scale.max(), f"grad_z at {n * T} rows: max error {err:.3e} vs term scale {scale.max():.3e}"


def _dense_dz_points(kind, Z, y, params, T, pts):
    """(d value / dz, the size of the summed terms) of points `pts` in the Kronecker form, from K built and factored in
    NumPy: only the K^-1 rows of those points' T rows are formed (O(N^2) memory beyond K)"""
    import scipy.linalg as sla
    from gpax_b200.mtgp import lcm_task_matrix
    from oracle import grad_oracle as gro
    from oracle import mtgp_oracle as mo
    n, d = Z.shape
    K = mo.lcm_cov(Z, Z, params, params["noise"], kind, True, T, JIT)
    cf = sla.cho_factor(K, lower=True)
    del K
    alpha = sla.cho_solve(cf, y)
    rows = np.array([p * T + t for p in pts for t in range(T)])
    E = np.zeros((n * T, rows.size))
    E[rows, np.arange(rows.size)] = 1.0
    Kinv = sla.cho_solve(cf, E).T                                        # [r, n T]
    aa = alpha[rows, None] * alpha[None, :]
    Wm = aa - Kinv
    Wm[np.arange(rows.size), rows] = 0.0
    Zr, t = np.repeat(Z, T, axis=0), np.tile(np.arange(T), n)
    Bs = lcm_task_matrix(params["W"], params["v"])
    g, sz = np.zeros((rows.size, d)), np.zeros((rows.size, d))
    for q in range(Bs.shape[0]):
        pq = {"k_length": params["k_length"][q], "k_scale": float(params["k_scale"][q]), "noise": 0.0}
        Dk = gro.kernel_dx(Zr[rows], Zr, pq, kind) * Bs[q][t[rows]][:, t][:, None, :]     # [r, d, n T]
        g += np.einsum("rj,rkj->rk", Wm, Dk)
        sz += np.einsum("rj,rkj->rk", np.abs(aa) + np.abs(Kinv), np.abs(Dk))
    return g.reshape(len(pts), T, d).sum(1), sz.reshape(len(pts), T, d).sum(1)


def test_device_and_host_pointers_agree(ctx):
    T, widths = 3, [16, 8, 2]
    X, task, y, layers, params = _problem(200, 10, widths, T, 2, 2, True, seed=3)
    theta, B, noise = _abi(params)
    flat = dko.flatten(layers)
    host = ctx.mtdkl_mll("RBF", X, task, y, widths, ACT["tanh"], flat, theta, B, noise, T, JIT, want_z=True)
    Xd, yd = ctx.to_device(X), ctx.to_device(y)
    try:
        dev = ctx.mtdkl_mll("RBF", Xd, task, yd, widths, ACT["tanh"], flat, theta, B, noise, T, JIT, want_z=True)
    finally:
        Xd.free()
        yd.free()
    assert host[0] == dev[0] and host[6] == dev[6]
    for a, b in zip(host[1:6], dev[1:6]):
        assert np.array_equal(a, b)


def test_indefinite_kernel_gives_nan(ctx):
    T, widths = 2, [16, 8, 2]
    X, task, y, layers, params = _problem(150, 10, widths, T, 1, 1, False, seed=4)
    theta, B, noise = _abi(params)
    noise = np.array([-5.0, 0.1])                      # negative noise: K is indefinite
    val, gt, gB, gn, gp, gz, info = ctx.mtdkl_mll("RBF", X, task, y, widths, ACT["relu"], dko.flatten(layers), theta, B, noise, 1,
                                                  JIT, want_z=True)
    assert info != 0
    for a in (gt, gB, gn, gp, gz):
        assert np.isnan(a).all()
    assert np.isnan(val)


def test_no_layers_gives_the_input_gradient(ctx):
    T = 3
    X, task, y, _, params = _problem(120, 3, [], T, 2, 2, True, seed=6)
    theta, B, noise = _abi(params)
    *_, gz, info = ctx.mtdkl_mll("Matern", X, task, y, [], ACT["relu"], np.zeros(0), theta, B, noise, T, JIT, want_z=True)
    assert info == 0
    _close(gz, mdo.lcm_dz("Matern", X, task, y, params, True, T, JIT)[4], 1e-8, "d/dX")


def test_refused_arguments(ctx):
    from gpax_b200._ffi import B200GPError
    X, task, y, layers, params = _problem(50, 10, [16, 8, 2], 2, 1, 1, False, seed=8)
    theta, B, noise = _abi(params)
    with pytest.raises(B200GPError):
        ctx.mtdkl_mll("Periodic", X, task, y, [16, 8, 2], 0, dko.flatten(layers), theta, B, noise)
    bad = task.copy()
    bad[3] = 2                                                  # outside [0, T)
    with pytest.raises(B200GPError):
        ctx.mtdkl_mll("RBF", X, bad, y, [16, 8, 2], 0, dko.flatten(layers), theta, B, noise)


# ---------------------------------------------------------------- viMTDKL
def _model_case(shared, L, seed, C=1):
    from gpax_b200 import viMTDKL
    T, D, n, P = 3, 6, 30, 8
    rng = np.random.default_rng(seed)
    X, Xn = rng.uniform(-1, 1, (n, D)), rng.uniform(-1, 1, (P, D))
    if shared:
        m = viMTDKL(D, 2, "Matern", num_latents=L, shared_input_space=True, num_tasks=T)
        tX, tN = np.tile(np.arange(T), n), np.tile(np.arange(T), P)
        Xin, Xnin = X, Xn
    else:
        m = viMTDKL(D, 2, "RBF", num_latents=L)
        tX, tN = np.arange(n) % T, rng.integers(0, T, P)
        Xin, Xnin = np.column_stack([X, tX]), np.column_stack([Xn, tN])
    rows = len(tX)
    Y = np.stack([np.cos(2 * np.repeat(X[:, 1], rows // n)) * (c + 1) + 0.2 * tX + 0.05 * rng.standard_normal(rows)
                  for c in range(C)])
    sets, kps = [], []
    for c in range(C):
        sets.append(_problem(2, D, [64, 64, 2], T, L, 2, shared, seed=seed + 10 + c)[3])
        p = _problem(2, D, [2], T, L, 2, shared, seed=seed + 20 + c)[4]
        kps.append({"k_length": p["k_length"], "k_scale": p["k_scale"].reshape(L, 1), "W": p["W"], "v": p["v"], "noise": p["noise"]})
    return m, Xin, Xnin, X, Xn, tX, tN, Y, sets, kps, T


def _oracle_params(kp):
    return dict(kp, k_scale=np.asarray(kp["k_scale"]).reshape(-1))


@pytest.mark.parametrize("shared", [False, True])
def test_vimtdkl_posterior_and_predict_match_oracle(shared):
    for L in (1, 2):
        m, Xin, Xnin, X, Xn, tX, tN, Y, sets, kps, T = _model_case(shared, L, seed=40 + L)
        kind = "Matern" if shared else "RBF"
        m.X_train, m.y_train = Xin, Y[0]
        nn = m.from_flat(dko.flatten(sets[0]))
        for noiseless in (False, True):
            mean, cov = m.get_mvn_posterior(Xnin, nn, kps[0], noiseless)
            rm, rc = mdo.posterior(kind, X, tX, Y[0], Xn, tN, sets[0], "relu", _oracle_params(kps[0]), shared, T, noiseless)
            _close(mean, rm, 1e-9, "mean")
            _close(cov, rc, 1e-9, "cov")
        m.nn_params, m.kernel_params = nn, kps[0]
        mean, var = m.predict(0, Xnin)
        rm, rc = mdo.posterior(kind, X, tX, Y[0], Xn, tN, sets[0], "relu", _oracle_params(kps[0]), shared, T)
        assert mean.shape == (len(Xn) * (T if shared else 1),)
        _close(mean, rm, 1e-9, "predict mean")
        _close(var, np.diag(rc), 1e-9, "predict var")
    # three channels: stacked leaves, one embedding and one posterior per channel
    m, Xin, Xnin, X, Xn, tX, tN, Y, sets, kps, T = _model_case(shared, 2, seed=50, C=3)
    m.X_train, m.y_train = Xin, Y
    m.nn_params = m.from_flat(np.stack([dko.flatten(s) for s in sets]))
    m.kernel_params = {k: np.stack([kp[k] for kp in kps]) for k in kps[0]}
    mean, var = m.predict(0, Xnin)
    assert mean.shape == var.shape == (3, len(Xn) * (T if shared else 1))
    for c in range(3):
        rm, rc = mdo.posterior("Matern" if shared else "RBF", X, tX, Y[c], Xn, tN, sets[c], "relu", _oracle_params(kps[c]), shared, T)
        _close(mean[c], rm, 1e-9, f"channel {c} mean")
        _close(var[c], np.diag(rc), 1e-9, f"channel {c} var")
    assert m.embed(Xnin).shape == (3, len(Xn), 2)


@pytest.mark.parametrize("shared", [False, True])
def test_vimtdkl_adam_matches_oracle(shared):
    """25 Adam steps of viMTDKL.fit from one fixed initialisation against the oracle's Adam on the same loss"""
    L, R = 2, 2
    m, Xin, _, X, _, tX, _, Y, sets, kps, T = _model_case(shared, L, seed=60)
    kp = kps[0]
    u0 = np.concatenate([np.log(kp["k_length"]).ravel(), np.ones(L), kp["W"].ravel(), np.log(kp["v"]).ravel(), np.log(kp["noise"])])
    flat0 = dko.flatten(sets[0])
    m._init_params = lambda r: (u0.copy(), flat0.copy())
    m.fit(0, Xin, Y[0], num_steps=25, step_size=5e-3, print_summary=False, progress_bar=False)
    nu = u0.size
    f = lambda p: mdo.vimtdkl_loss(m._fused, X, tX, Y[0], p[:nu], p[nu:], 6, [64, 64, 2], "relu", L, T, R, shared)  # noqa: E731
    ref, _ = dko.adam(f, np.concatenate([u0, flat0]), 25, 5e-3)
    np.testing.assert_allclose(m.loss, ref, rtol=1e-7)
    assert set(m.kernel_params) == {"k_length", "k_scale", "W", "v", "noise"}
    assert m.kernel_params["k_scale"].shape == (L, 1) and m.kernel_params["W"].shape == (L, T, R)


# ---------------------------------------------------------------- the reference's tests/test_vimtdkl.py, in form
def _dummy(rng):
    return rng.standard_normal((21, 36)), rng.standard_normal(21)


@pytest.mark.parametrize("num_latents", [1, 2])
@pytest.mark.parametrize("num_tasks", [2, 3])
@pytest.mark.parametrize("data_kernel", ["RBF", "Matern"])
def test_fit_multitask(data_kernel, num_tasks, num_latents):
    from gpax_b200 import viMTDKL
    rng = np.random.default_rng(0)
    X, y = _dummy(rng)
    X = np.column_stack([X, rng.integers(0, num_tasks, len(X))])
    m = viMTDKL(X.shape[-1] - 1, 2, data_kernel, num_latents=num_latents, shared_input_space=False)
    m.fit(0, X, y, num_steps=10, print_summary=False, progress_bar=False)
    assert isinstance(m.kernel_params, dict) and isinstance(m.nn_params, dict)
    assert np.isfinite(m.loss).all()


@pytest.mark.parametrize("num_latents", [1, 2])
@pytest.mark.parametrize("num_tasks", [2, 3])
@pytest.mark.parametrize("data_kernel", ["RBF", "Matern"])
def test_fit_multitask_shared_input(data_kernel, num_tasks, num_latents):
    from gpax_b200 import viMTDKL
    rng = np.random.default_rng(1)
    X, y = _dummy(rng)
    y = np.repeat(y[:, None], num_tasks, axis=1).reshape(-1)
    m = viMTDKL(X.shape[-1], 2, data_kernel, num_latents=num_latents, shared_input_space=True, num_tasks=num_tasks)
    m.fit(0, X, y, num_steps=10, print_summary=False, progress_bar=False)
    assert isinstance(m.kernel_params, dict) and isinstance(m.nn_params, dict)
    assert np.isfinite(m.loss).all()


@pytest.mark.parametrize("num_latents", [1, 2])
@pytest.mark.parametrize("num_tasks", [2, 3])
@pytest.mark.parametrize("data_kernel", ["RBF", "Matern"])
def test_fit_predict_multitask(data_kernel, num_tasks, num_latents):
    from gpax_b200 import viMTDKL
    rng = np.random.default_rng(2)
    X, y = _dummy(rng)
    X = np.column_stack([X, rng.integers(0, num_tasks, len(X))])
    m = viMTDKL(X.shape[-1] - 1, 2, data_kernel, num_latents=num_latents, shared_input_space=False)
    m.fit(0, X, y, num_steps=10, print_summary=False, progress_bar=False)
    X_test, _ = _dummy(rng)
    X_test = np.column_stack([X_test, np.ones(len(X_test))])
    mean, var = m.predict(0, X_test)
    assert len(mean) == len(X_test) and len(var) == len(X_test)
    assert np.isfinite(mean).all() and np.isfinite(var).all()


def test_w_leaves_its_initial_value():
    from gpax_b200 import viMTDKL
    rng = np.random.default_rng(3)
    X = np.column_stack([rng.uniform(-1, 1, (40, 5)), np.arange(40) % 3])
    y = np.sin(2 * X[:, 0]) + 0.5 * X[:, -1]
    m = viMTDKL(5, num_latents=2)
    m.X_train = X
    u0, _ = m._init_params(np.random.default_rng(0))
    W0 = m._theta(u0)["W"]
    m.fit(0, X, y, num_steps=20, print_summary=False, progress_bar=False)
    assert m.kernel_params["W"].shape == W0.shape
    assert np.abs(m.kernel_params["W"] - W0).max() > 1e-3


def test_acquisitions_on_a_fitted_model_use_the_embedding():
    from gpax_b200 import acquisition
    m, Xin, Xnin, X, Xn, tX, tN, Y, sets, kps, T = _model_case(False, 2, seed=70)
    m.fit(0, Xin, Y[0], num_steps=5, print_summary=False, progress_bar=False)
    mean, var = m.predict(0, Xnin)
    layers = [(m.nn_params[n]["w"], m.nn_params[n]["b"]) for n in ("mlp/~/linear", "mlp/~/linear_1", "mlp/~/linear_2")]
    rm, rc = mdo.posterior("RBF", X, tX, Y[0], Xn, tN, layers, "relu", _oracle_params(m.kernel_params), False, T)
    _close(mean, rm, 1e-9, "mean")
    _close(var, np.diag(rc), 1e-9, "var")
    ucb = acquisition.UCB(0, m, Xnin, beta=0.5)
    ei = acquisition.EI(0, m, Xnin)
    np.testing.assert_allclose(ucb, m.ctx.acq_moments("UCB", mean, var, None, 0.5, False), rtol=1e-12)
    np.testing.assert_allclose(ei, m.ctx.acq_moments("EI", mean, var, None, 0.0, False), rtol=1e-12)
    out = m._posterior_batched(Xnin, m.get_samples(), False, False, ("mean", "var"))
    _close(out["mean"][0], rm, 1e-9, "seam mean")
    with pytest.raises(NotImplementedError):
        m._posterior_grad(Xnin[:1], m.get_samples(), False, False)


# ---------------------------------------------------------------- against the reference's own vi_mtdkl.py
@pytest.mark.parametrize("tag", ["mt_L1", "mt_L2", "kron_L1", "kron_L2"])
def test_vimtdkl_matches_golden(tag):
    import os
    from gpax_b200 import viMTDKL
    G = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_mtdkl.npz"))
    shared, L = tag.startswith("kron"), int(tag[-1])
    m = viMTDKL(6, 2, "RBF" if shared else "Matern", num_latents=L, shared_input_space=shared, num_tasks=3 if shared else None,
                rank=2)
    m.X_train, m.y_train = G[tag + "_X"], G[tag + "_y"]
    nn = {n: {"w": G[f"{tag}_{n}_w"], "b": G[f"{tag}_{n}_b"]} for n in ("mlp/~/linear", "mlp/~/linear_1", "mlp/~/linear_2")}
    kp = {k: G[f"{tag}_p_{k}"] for k in ("k_length", "k_scale", "W", "v", "noise")}
    for nl in (False, True):
        mean, cov = m.get_mvn_posterior(G[tag + "_X_new"], nn, kp, nl)
        _close(mean, G[f"{tag}_mean_noiseless{int(nl)}"], 1e-9, "mean")
        _close(cov, G[f"{tag}_cov_noiseless{int(nl)}"], 1e-9, "cov")
    m.nn_params, m.kernel_params = nn, kp
    mean, var = m.predict(0, G[tag + "_X_new"])
    _close(mean, G[tag + "_predict_mean"], 1e-9, "predict mean")
    _close(var, G[tag + "_predict_var"], 1e-9, "predict var")


# ---------------------------------------------------------------- KG and the q-batch functions
def _brute_force_kg(kind, X, tX, y, Xn, tN, layers, p, T, ysim, noiseless, maximize):
    """the reference's kg (base_acq.py:158-232): for every candidate c and simulation i, the posterior mean over the
    candidates after appending (x_c, task_c, ysim[i, c]) to the training data, re-inverted from scratch"""
    mean, _ = mdo.posterior(kind, X, tX, y, Xn, tN, layers, "relu", p, False, T, noiseless)
    best = mean.max() if maximize else mean.min()
    out = np.zeros(len(Xn))
    for c in range(len(Xn)):
        for ys in ysim:
            ma, _ = mdo.posterior(kind, np.vstack([X, Xn[c]]), np.r_[tX, tN[c]], np.r_[y, ys[c]], Xn, tN, layers, "relu", p, False, T,
                                  noiseless)
            u = (ma.max() if maximize else ma.min()) - best
            out[c] += (u if maximize else -u) / len(ysim)
    return out


@pytest.mark.parametrize("noiseless,maximize", [(True, True), (False, False)])
def test_kg_matches_the_reference_update_with_a_noise_per_task(noiseless, maximize):
    from gpax_b200 import acquisition
    m, Xin, Xnin, X, Xn, tX, tN, Y, sets, kps, T = _model_case(False, 2, seed=80)
    kp = dict(kps[0], noise=np.array([0.02, 0.1, 0.3]))           # distinct noise per task
    m.X_train, m.y_train = Xin, Y[0]
    m.nn_params, m.kernel_params = m.from_flat(dko.flatten(sets[0])), kp
    n = 3
    eps = np.random.default_rng(1).standard_normal((n, len(Xn)))
    sample = m.get_samples()
    got = acquisition.kg(m, Xnin, sample, n=n, maximize=maximize, noiseless=noiseless, eps=eps)
    ysim = m._posterior_batched(Xnin, sample, False, noiseless, ("mean",), eps=eps.reshape(1, n, -1))["y_sampled"][0]
    ref = _brute_force_kg("RBF", X, tX, Y[0], Xn, tN, sets[0], _oracle_params(kp), T, ysim, noiseless, maximize)
    mean, _ = mdo.posterior("RBF", X, tX, Y[0], Xn, tN, sets[0], "relu", _oracle_params(kp), False, T, noiseless)
    err = np.abs(got - ref).max()
    assert err <= 1e-8 * np.abs(mean).max(), f"kg: max error {err:.3e} vs mean scale {np.abs(mean).max():.3e}"
    kg_all = acquisition.KG(0, m, Xnin, n=2)
    assert kg_all.shape == (len(Xn),) and np.isfinite(kg_all).all()


def test_kg_refused_in_the_kronecker_form_and_q_batch_needs_a_bayesian_model():
    from gpax_b200 import acquisition
    m, Xin, Xnin, X, Xn, tX, tN, Y, sets, kps, T = _model_case(True, 2, seed=90)
    m.X_train, m.y_train = Xin, Y[0]
    m.nn_params, m.kernel_params = m.from_flat(dko.flatten(sets[0])), kps[0]
    with pytest.raises(NotImplementedError, match="Kronecker"):
        acquisition.KG(0, m, Xnin, n=2)
    m2, Xin2, Xnin2, *_ = _model_case(False, 1, seed=91)
    m2.fit(0, Xin2, _model_case(False, 1, seed=91)[7][0], num_steps=2, print_summary=False, progress_bar=False)
    with pytest.raises(ValueError, match="fully Bayesian"):
        acquisition.qEI(0, m2, Xnin2, subsample_size=2)
