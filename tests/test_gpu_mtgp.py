"""GPU: MultiTaskGP / CoregGP -- b2gp_posterior_multitask and b2gp_mll_multitask against oracle/mtgp_oracle.py."""
import numpy as np
import pytest

from oracle import mtgp_oracle as mo

pytestmark = pytest.mark.gpu


def params(rng, L, T, R, d, kind, S=None):
    sh = () if S is None else (S,)
    p = {"k_length": rng.uniform(0.4, 0.9, sh + (L, d)), "k_scale": rng.uniform(0.8, 1.3, sh + (L,)),
         "W": rng.normal(0, 0.7, sh + (L, T, R)), "v": rng.uniform(0.3, 0.8, sh + (L, T)), "noise": rng.uniform(0.05, 0.2, sh + (T,)),
         "period": rng.uniform(1.5, 2.5, sh + (L,)) if kind == "Periodic" else None}
    return p


def data(rng, n, d, T, shared):
    X = rng.uniform(0, 2, (n, d))
    if not shared:
        X = np.c_[X, rng.integers(0, T, n)]
    y = rng.standard_normal(n * T if shared else n)
    return X, y


def draw(p, s):
    return {k: (None if v is None else np.asarray(v)[s]) for k, v in p.items()}


def packed(p, L, T, d, S):
    th = np.empty((S, L, d + 2))
    th[..., :d] = p["k_length"]
    th[..., d] = p["k_scale"]
    th[..., d + 1] = 1.0 if p["period"] is None else p["period"]
    B = np.einsum("sltr,slur->sltu", p["W"], p["W"]) + p["v"][..., None] * np.eye(T)
    return th, B, p["noise"]


def run_post(ctx, kind, X, y, Xn, p, L, T, d, S, shared, noiseless=False, want=("mean", "var", "cov"), eps=None):
    Xd, tt, g = mo.expand(X, shared, T)
    Xnd, tn, _ = mo.expand(Xn, shared, T)
    th, B, nz = packed(p, L, T, d, S)
    return ctx.posterior_multitask(kind, Xd, tt, y, Xnd, tn, th, B, nz, g, noiseless, 1e-6, want, eps)


def tol(K):
    return max(1e-9, 1e-15 * np.linalg.cond(K))


CASES = [  # kind, shared, L, T, N points, noiseless
    ("Matern", False, 2, 3, 300, False),
    ("Matern", False, 2, 3, 300, True),
    ("RBF", True, 2, 2, 150, False),
    ("Periodic", False, 1, 3, 280, False),
    ("RBF", False, 1, 3, 290, False),   # CoregGP's shape
]


@pytest.mark.parametrize("kind,shared,L,T,n,noiseless", CASES)
@pytest.mark.parametrize("route", ["rec", "tall"])
def test_posterior_vs_oracle(kind, shared, L, T, n, noiseless, route):
    import gpax_b200
    rng = np.random.default_rng(n + L)
    d, S, P = 2, 3, 40
    if route == "tall":
        n = 2500 // T if shared else 2500
    X, y = data(rng, n, d, T, shared)
    Xn, _ = data(rng, P if not shared else P // T, d, T, shared)
    Xn[: min(len(Xn), 5)] = X[:5]                        # some test inputs coincide with training inputs
    p = params(rng, L, T, 2, d, kind, S)
    ctx = gpax_b200.Context(streams=2)
    with ctx.options(ozaki=0 if route == "rec" else 7):
        before = ctx.path_counts()["potrf_tall"]
        out = run_post(ctx, kind, X, y, Xn, p, L, T, d, S, shared, noiseless)
        tall = ctx.path_counts()["potrf_tall"] - before
    assert tall == (S if route == "tall" else 0)
    assert (out["info"] == 0).all()
    for s in range(S):
        ps = draw(p, s)
        m_ref, c_ref = mo.posterior(X, y, Xn, ps, kind, shared, T, noiseless)
        K = mo.lcm_cov(X, X, ps, np.asarray(ps["noise"]), kind, shared, T)
        t = tol(K)
        np.testing.assert_allclose(out["mean"][s], m_ref, rtol=t, atol=t * np.abs(m_ref).max())
        np.testing.assert_allclose(out["cov"][s], c_ref, rtol=t, atol=t * np.abs(c_ref).max())
        np.testing.assert_allclose(out["var"][s], np.diag(c_ref), rtol=t, atol=t * np.abs(c_ref).max())
    ctx.close()


def test_samples_are_mean_plus_chol_cov_eps():
    import gpax_b200
    rng = np.random.default_rng(3)
    L, T, d, S = 2, 3, 2, 2
    X, y = data(rng, 120, d, T, False)
    Xn, _ = data(rng, 30, d, T, False)
    p = params(rng, L, T, 2, d, "RBF", S)
    eps = rng.standard_normal((S, 4, 30))
    ctx = gpax_b200.default_context()
    out = run_post(ctx, "RBF", X, y, Xn, p, L, T, d, S, False, want=("mean", "cov"), eps=eps)
    for s in range(S):
        ref = out["mean"][s] + eps[s] @ np.linalg.cholesky(out["cov"][s]).T
        np.testing.assert_allclose(out["y_sampled"][s], ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())


@pytest.mark.parametrize("kind,shared,L,T,n,route", [("Matern", False, 2, 3, 300, "rec"), ("RBF", True, 2, 2, 150, "rec"),
                                                     ("Periodic", False, 1, 2, 250, "rec"), ("RBF", False, 2, 3, 2500, "rec"),
                                                     ("RBF", False, 2, 3, 2500, "tall"), ("Matern", True, 2, 2, 1250, "tall")])
def test_mll_vs_oracle(kind, shared, L, T, n, route):
    import gpax_b200
    rng = np.random.default_rng(n)
    d = 2
    X, y = data(rng, n, d, T, shared)
    p = params(rng, L, T, 2, d, kind)
    th, B, nz = (a[0] for a in packed({k: (None if v is None else np.asarray(v)[None]) for k, v in p.items()}, L, T, d, 1))
    Xd, tt, g = mo.expand(X, shared, T)
    ctx = gpax_b200.default_context()
    with ctx.options(ozaki=0 if route == "rec" else 7):
        before = ctx.path_counts()["potrf_tall"]
        val, gt, gB, gn, alpha, info = ctx.mll_multitask(kind, Xd, tt, y, th, B, nz, g, want_alpha=True)
        assert ctx.path_counts()["potrf_tall"] - before == (1 if route == "tall" else 0)
        again = ctx.mll_multitask(kind, Xd, tt, y, th, B, nz, g, want_alpha=True)
    assert info == 0
    rv, rt, rB, rn = mo.loglik_grad(X, y, p, kind, shared, T)
    assert abs(val - rv) <= 1e-9 * abs(rv)
    scale = max(np.abs(rt).max(), np.abs(rB).max(), np.abs(rn).max())
    used = slice(None) if kind == "Periodic" else slice(0, d + 1)
    np.testing.assert_allclose(gt[:, used], rt[:, used], rtol=1e-6, atol=1e-7 * scale)
    np.testing.assert_allclose(gB, rB, rtol=1e-6, atol=1e-7 * scale)
    np.testing.assert_allclose(gn, rn, rtol=1e-6, atol=1e-7 * scale)
    # determinism: identical calls, identical bits
    assert again[0] == val and (again[1] == gt).all() and (again[2] == gB).all() and (again[3] == gn).all()
    assert (again[4] == alpha).all()


def test_not_positive_definite_gives_nan():
    import gpax_b200
    rng = np.random.default_rng(5)
    L, T, d = 1, 2, 1
    X, y = data(rng, 60, d, T, False)
    p = params(rng, L, T, 1, d, "RBF", 1)
    p["W"][:] = 0.0
    p["v"][:] = -1.0
    p["noise"][:] = 0.0
    ctx = gpax_b200.default_context()
    out = run_post(ctx, "RBF", X, y, X[:10], p, L, T, d, 1, False)
    assert out["info"][0] > 0 and np.isnan(out["mean"]).all() and np.isnan(out["var"]).all() and np.isnan(out["cov"]).all()
    th, B, nz = (a[0] for a in packed(p, L, T, d, 1))
    Xd, tt, g = mo.expand(X, False, T)
    val, gt, gB, gn, _, info = ctx.mll_multitask("RBF", Xd, tt, y, th, B, nz, g)
    assert info > 0 and np.isnan(val) and np.isnan(gt).all() and np.isnan(gB).all() and np.isnan(gn).all()


def test_refusals():
    import gpax_b200
    from gpax_b200 import _ffi
    rng = np.random.default_rng(6)
    ctx = gpax_b200.default_context()

    def call(T=2, L=1, d=2, task=None, flags=0):
        X = rng.uniform(0, 1, (20, d))
        t = np.arange(20) % T if task is None else task
        p = params(rng, L, T, 1, d, "RBF", 1)
        th, B, nz = packed(p, L, T, d, 1)
        return ctx.posterior_multitask("RBF", X, t, np.ones(20), X[:4], t[:4], th, B, nz, flags=flags)

    call()
    for kw in ({"T": 9}, {"L": 5}, {"d": 17}, {"task": np.r_[np.zeros(19, int), 2]}, {"task": np.r_[np.zeros(19, int), -1]},
               {"flags": _ffi.FLAG_DEVICE_PTRS}, {"flags": _ffi.FLAG_F32}):
        launches = ctx.last_timing()["launches"]
        with pytest.raises(gpax_b200.B200GPError):
            call(**kw)
        assert ctx.last_timing()["launches"] == launches
    with pytest.raises(gpax_b200.B200GPError):
        X = rng.uniform(0, 1, (20, 2))
        ctx.mll_multitask("RBF", X, np.full(20, 3), np.ones(20), np.ones((1, 4)), np.eye(2)[None], np.ones(2))


def test_multitask_call_leaves_the_factor_cache_invalid():
    import gpax_b200
    rng = np.random.default_rng(7)
    N, d = 300, 2
    X = rng.uniform(0, 1, (N, d))
    y = rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (20, d))
    theta = np.array([[0.5, 0.6, 1.1, 0.1, 1.0]])
    ctx = gpax_b200.Context()
    ctx.posterior("Matern", X, y, Xn, theta, want=("mean", "var"))
    Xm, ym = data(rng, N, d, 3, False)
    p = params(rng, 2, 3, 2, d, "Matern", 1)
    run_post(ctx, "Matern", Xm, ym, Xm[:20], p, 2, 3, d, 1, False)
    hits = ctx.cache_hits()
    got = ctx.posterior("Matern", X, y, Xn, theta, want=("mean", "var"))
    assert ctx.cache_hits() == hits
    fresh = gpax_b200.Context().posterior("Matern", X, y, Xn, theta, want=("mean", "var"))
    assert (got["mean"] == fresh["mean"]).all() and (got["var"] == fresh["var"]).all()


# ---------------------------------------------------------------------------------------------- models
def dummy_data(T, shared, n=8, seed=0):
    rng = np.random.default_rng(seed)
    X = np.linspace(0, 1, n)[:, None]
    if shared:
        y = np.repeat(np.sin(6 * X[:, 0])[:, None], T, axis=1).reshape(-1) + 0.05 * rng.standard_normal(n * T)
        return X, y
    Xt = np.concatenate([np.c_[X, np.full(n, t)] for t in range(T)])
    return Xt, np.sin(6 * Xt[:, 0]) + 0.1 * Xt[:, 1] + 0.05 * rng.standard_normal(len(Xt))


def mean_fn(x, p):
    return p["a"] * x[:, 0]


def mean_fn_prior():
    from gpax_b200 import priors as numpyro
    return {"a": numpyro.sample("a", numpyro.distributions.Normal(0, 1))}


# the reference's matrix (tests/test_mtgp.py) for the multitask form; one case per kernel for the Kronecker form, whose fit
# differs only in the row expansion
FIT_CASES = [(k, T, L, False) for k in ("RBF", "Matern", "Periodic") for T in (2, 3) for L in (1, 2)] + \
    [("RBF", 2, 2, True), ("Matern", 3, 1, True), ("Periodic", 2, 2, True)]


@pytest.mark.parametrize("kind,T,L,shared", FIT_CASES)
def test_multitaskgp_fit(kind, T, L, shared):
    import gpax_b200
    X, y = dummy_data(T, shared)
    m = gpax_b200.MultiTaskGP(1, kind, num_latents=L, shared_input_space=shared, num_tasks=T if shared else None)
    m.fit(0, X, y, num_warmup=50, num_samples=50, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert s["k_length"].shape == (50, L, 1) and s["W"].shape == (50, L, T, T - 1)     # site values, before the squeeze
    assert s["v"].shape == (50, L, T) and s["noise"].shape == (50, T) and s["k_scale"].shape == (50, L)
    if kind == "Periodic":
        assert s["period"].shape == (50, L, 1)
    Xn = X[:3]
    mean, ys = m.predict(1, Xn, n=2)
    P = 3 * T if shared else 3
    assert mean.shape == (P,) and ys.shape == (50, 2, P) and np.isfinite(ys).all()


@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
@pytest.mark.parametrize("T", [2, 3])
def test_coreggp_fit_and_predict_vs_oracle(kind, T):
    import gpax_b200
    X, y = dummy_data(T, False)
    m = gpax_b200.CoregGP(1, kind, rank=1, mean_fn=mean_fn, mean_fn_prior=mean_fn_prior)
    m.fit(0, X, y, num_warmup=50, num_samples=50, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert s["k_length"].shape == (50, 1) and s["W"].shape == (50, T, 1) and s["v"].shape == (50, T) and s["noise"].shape == (50, T)
    assert s["a"].shape == (50,) and s["k_scale"].shape == (50,)
    Xn = X[::3]
    sub = {k: v[:5] for k, v in s.items()}
    mean, _ = m.predict(2, Xn, sub, n=1)
    ref = []
    for i in range(5):
        ps = {"k_length": sub["k_length"][i][None], "k_scale": np.ones(1), "W": sub["W"][i][None], "v": sub["v"][i][None],
              "noise": sub["noise"][i], "period": sub["period"][i].reshape(1) if kind == "Periodic" else None}
        mu, _ = mo.posterior(X, y - sub["a"][i] * X[:, 0], Xn, ps, kind, False)
        ref.append(mu + sub["a"][i] * Xn[:, 0])
    np.testing.assert_allclose(mean, np.mean(ref, 0), rtol=1e-8, atol=1e-9)


def test_log_joint_gradient_matches_differences():
    import gpax_b200
    from gpax_b200.inference import MTLogJoint
    X, y = dummy_data(3, False, n=10)
    m = gpax_b200.MultiTaskGP(1, "Matern", num_latents=2, mean_fn=mean_fn, mean_fn_prior=mean_fn_prior)
    m.X_train, m.y_train = X, y
    lj = MTLogJoint(m)
    rng = np.random.default_rng(9)
    for _ in range(3):
        u = lj.init_u() + 0.3 * rng.standard_normal(lj.dim)
        val, g = lj(u, jacobian=True)
        h = 1e-5
        for k in range(lj.dim):
            e = np.zeros(lj.dim)
            e[k] = h
            num = (lj(u + e, True)[0] - lj(u - e, True)[0]) / (2 * h)
            assert abs(g[k] - num) <= 1e-4 * max(1.0, abs(num)), (k, g[k], num)


def test_ei_on_coreggp_equals_ei_of_oracle_moments():
    """acquisition.EI on a fitted CoregGP: the moments of the oracle's predictive draws, mean + chol(cov) eps with the eps
    predict draws, through the reference's EI formula (oracle/acq_oracle.py)"""
    import gpax_b200
    from gpax_b200 import acquisition
    from gpax_b200.gp import _eps_dtype
    from gpax_b200.utils import posterior_eps
    from oracle import acq_oracle
    X, y = dummy_data(2, False)
    m = gpax_b200.CoregGP(1, "RBF")
    m.fit(0, X, y, num_warmup=50, num_samples=50, progress_bar=False, print_summary=False)
    s = m.get_samples()
    Xn = X[1::2]
    got = np.asarray(acquisition.EI(3, m, Xn))
    S, P = len(s["W"]), len(Xn)
    eps = np.asarray(posterior_eps(3, S, 1, P, _eps_dtype()), dtype=np.float64).reshape(S, 1, P)
    ys = []
    for i in range(S):
        ps = {"k_length": s["k_length"][i][None], "k_scale": np.ones(1), "W": s["W"][i][None], "v": s["v"][i][None],
              "noise": s["noise"][i], "period": None}
        mu, cov = mo.posterior(X, y, Xn, ps, "RBF", False)
        ys.append(mu + eps[i] @ np.linalg.cholesky(cov).T)
    ref = acq_oracle.ei(*acq_oracle.moments_from_samples(np.stack(ys)))
    np.testing.assert_allclose(got, ref, rtol=1e-7, atol=1e-9 * np.abs(ref).max())


GOLDEN = {"mt_matern_nl0": ("Matern", False, 2, 3), "mt_matern_nl1": ("Matern", False, 2, 3), "kron_rbf": ("RBF", True, 2, 2),
          "mt_periodic": ("Periodic", False, 1, 3), "coreg_rbf": ("RBF", False, 1, 3), "coreg_rbf_pn": ("RBF", False, 1, 3)}


@pytest.mark.parametrize("tag", sorted(GOLDEN))
def test_get_mvn_posterior_matches_the_reference(tag):
    """the public get_mvn_posterior against the reference's own get_mvn_posterior (reference_vectors_mt.npz)"""
    import os
    import gpax_b200
    gm = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_mt.npz"))
    kind, shared, L, T = GOLDEN[tag]
    X, d = gm[tag + "_X"], gm[tag + "_Xnew"].shape[1] - (0 if shared else 1)
    if tag.startswith("coreg"):
        m = gpax_b200.CoregGP(d, kind)
    else:
        m = gpax_b200.MultiTaskGP(d, kind, num_latents=L, shared_input_space=shared, num_tasks=T)
    m.X_train, m.y_train = X, gm[tag + "_y"]
    p = {k[len(tag) + 3:]: gm[k] for k in gm.files if k.startswith(tag + "_p_")}
    mean, cov = m.get_mvn_posterior(gm[tag + "_Xnew"], p, noiseless=tag.endswith("nl1"))
    np.testing.assert_allclose(mean, gm[tag + "_mean"], rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(cov, gm[tag + "_cov"], rtol=1e-9, atol=1e-10)


def test_sample_from_prior_leaves_the_model_untouched():
    import gpax_b200
    X, _ = dummy_data(3, False)
    m = gpax_b200.CoregGP(1, "RBF")
    ys = m.sample_from_prior(0, X, num_samples=3)
    assert ys.shape == (3, len(X)) and np.isfinite(ys).all() and m.X_train is None
