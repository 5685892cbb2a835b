"""b2gp_mll_batch on the GPU: every member against the NumPy oracle on both routes, the route counter and launch count,
bit-identity of the large route with b2gp_mll / b2gp_dkl_mll(n_layers = 0), isolation of a non-positive-definite member,
determinism, the refusals, and vExactGP / UIGP fitted end to end."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import oracle.dkl_oracle as dko
import oracle.fit_oracle as fo

pytestmark = pytest.mark.gpu

KINDS = ["RBF", "Matern", "Periodic"]
JIT = 1e-6
# the bound of the one-launch route, as include/b200gp.h states it
SMALL_MAX = int(re.search(r"#define B2GP_MLL_BATCH_SMALL_MAX_N (\d+)",
                          open(os.path.join(os.path.dirname(__file__), "..", "include", "b200gp.h")).read()).group(1))


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def batch_problem(kind, B, N, d, seed):
    """B members with their own inputs, targets and hyper-parameters"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (B, N, d))
    y = np.sin(4 * X[..., 0]) + 0.2 * rng.standard_normal((B, N))
    ell = rng.uniform(0.25, 0.6, (B, d)) * np.sqrt(d)
    theta = np.concatenate([ell, rng.uniform(0.8, 1.5, (B, 1)), rng.uniform(0.05, 0.2, (B, 1)),
                            (rng.uniform(0.6, 1.0, (B, 1)) if kind == "Periodic" else np.ones((B, 1)))], axis=1)
    return X, y, theta


def cond_of(kind, X, theta):
    k, _ = fo._derivs(X, theta, kind)
    return float(np.linalg.cond(k + (theta[X.shape[1] + 1] + JIT) * np.eye(len(X))))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", [1, 3, 16])
@pytest.mark.parametrize("N", sorted({1, 2, 31, 64, 127, 128, 129, 300, SMALL_MAX, SMALL_MAX + 1}))
@pytest.mark.parametrize("B", [1, 3, 200])
def test_members_match_the_oracle(ctx, kind, d, N, B):
    if B == 200 and N > SMALL_MAX:
        pytest.skip("the large route is a loop over b2gp_mll, covered member by member at B = 1 and 3")
    X, y, theta = batch_problem(kind, B, N, d, seed=1000 * d + N + B)
    val, g, alpha, gx, info = ctx.mll_batch(kind, X, y, theta, JIT, True, True, True)
    assert (info == 0).all()
    # at B = 200 (more than one wave of CTAs on 132 SMs) every 7th member and the last one are checked: the host oracle
    # dominates the test's time
    for b in (range(B) if B < 200 else list(range(0, B, 7)) + [B - 1]):
        t = fo.tau(cond_of(kind, X[b], theta[b]))
        rv, rg, ra, _, sg = fo.mll_grad(kind, X[b], y[b], theta[b], JIT)
        _, _, rgx, sgx = dko.mll_dz(kind, X[b], y[b], theta[b], JIT)
        assert fo.err_ratio([val[b]], [rv], [abs(rv) + N], t) <= 1, f"value, member {b}"
        assert fo.err_ratio(g[b], rg, sg, t) <= 1, f"grad, member {b}"
        assert fo.err_ratio(gx[b], rgx, sgx, t) <= 1, f"grad_x, member {b}"
        np.testing.assert_allclose(alpha[b], ra, rtol=0, atol=t * np.abs(ra).max() * 10)


@pytest.mark.parametrize("N, small", [(SMALL_MAX // 2, True), (SMALL_MAX, True), (SMALL_MAX + 1, False), (128, SMALL_MAX >= 128)])
def test_route_counter_and_launch_count(ctx, N, small):
    launches = []
    for B in (1, 200):
        X, y, theta = batch_problem("RBF", B, N, 2, seed=N)
        c0 = ctx.path_counts()["mll_batch_small"]
        ctx.mll_batch("RBF", X, y, theta, JIT, True, False, True)
        assert ctx.path_counts()["mll_batch_small"] - c0 == int(small)
        launches.append(ctx.last_timing()["launches"])
    if small:
        assert launches[0] == launches[1] == 1


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("N", [SMALL_MAX + 1, 300])
def test_large_route_is_bit_identical_to_the_single_member_calls(ctx, kind, N):
    X, y, theta = batch_problem(kind, 3, N, 3, seed=N + 7)
    val, g, alpha, gx, info = ctx.mll_batch(kind, X, y, theta, JIT, True, True, True)
    for b in range(3):
        mv, mg, ma, minfo = ctx.mll(kind, X[b], y[b], theta[b], JIT, True, True)
        dv, dg, _, dgx, dinfo = ctx.dkl_mll(kind, X[b], y[b], [], 0, np.zeros(0), theta[b], JIT, want_params=False, want_z=True)
        assert info[b] == minfo == dinfo == 0
        assert val[b] == mv == dv
        assert np.array_equal(g[b], mg) and np.array_equal(g[b], dg)
        assert np.array_equal(alpha[b], ma) and np.array_equal(gx[b], dgx)


@pytest.mark.parametrize("N", [SMALL_MAX // 2, 200])
def test_a_non_pd_member_touches_only_its_own_outputs(ctx, N):
    X, y, theta = batch_problem("Matern", 5, N, 2, seed=N)
    bad = theta.copy()
    bad[2, 3] = -50.0                                          # a negative noise variance: K is not positive definite
    val, g, alpha, gx, info = ctx.mll_batch("Matern", X, y, bad, JIT, True, True, True)
    assert info[2] != 0 and np.isnan(val[2]) and np.isnan(g[2]).all() and np.isnan(alpha[2]).all() and np.isnan(gx[2]).all()
    keep = [0, 1, 3, 4]
    rv, rg, ra, rgx, rinfo = ctx.mll_batch("Matern", X[keep], y[keep], theta[keep], JIT, True, True, True)
    assert (info[keep] == 0).all() and (rinfo == 0).all()
    assert np.array_equal(val[keep], rv) and np.array_equal(g[keep], rg)
    assert np.array_equal(alpha[keep], ra) and np.array_equal(gx[keep], rgx)


@pytest.mark.parametrize("N, B", [(SMALL_MAX - 5, 50), (200, 2)])
def test_identical_calls_give_identical_bits(ctx, N, B):
    X, y, theta = batch_problem("Periodic", B, N, 3, seed=3)
    a = ctx.mll_batch("Periodic", X, y, theta, JIT, True, True, True)
    b = ctx.mll_batch("Periodic", X, y, theta, JIT, True, True, True)
    for u, v in zip(a, b):
        assert np.array_equal(u, v)


def test_refusals(ctx):
    from gpax_b200 import _ffi
    lib = ctx.lib
    B, N = 2, 16

    def call(kind=0, d=2, flags=0, grad=True, gx=False):
        X, y, th = np.zeros((B, N, d)), np.zeros((B, N)), np.ones((B, d + 3))
        val, g, x = np.zeros(B), np.zeros((B, d + 3)), np.zeros((B, N, d))
        info = np.zeros(B, dtype=np.int32)
        p = lambda a: C.c_void_p(a.ctypes.data)     # noqa: E731
        return lib.b2gp_mll_batch(ctx.h, kind, p(X), N, p(y), d, B, p(th), JIT, flags, p(val), p(g) if grad else None, None,
                                  p(x) if gx else None, p(info))
    assert call(kind=3) == call(kind=4) == -4                  # NNGP kinds: B2GP_ERR_UNSUPPORTED
    assert call(flags=_ffi.FLAG_F32) == -4
    assert call(flags=_ffi.FLAG_DEVICE_PTRS) == -4
    assert call(d=17) == -1                                    # B2GP_ERR_ARG
    assert call(grad=False, gx=True) == -1
    assert call() == 0
    with pytest.raises(ValueError):
        ctx.mll_batch("RBF", np.zeros((2, 4, 1)), np.zeros((2, 4)), np.ones((2, 3)))


# ------------------------------------------------------------------ the models end to end
def dummy_data(seed=0):
    """the reference's tests/test_vgp.py:15-23 data: 3 tasks of 8 points in [1, 2]"""
    rng = np.random.default_rng(seed)
    X = np.array([np.linspace(1, 2, 8) + 0.1 * rng.standard_normal(8) for _ in range(3)])
    return X, 10 * X ** 2


@pytest.mark.parametrize("kernel", ["RBF", "Periodic"])
def test_vexact_fit_predict_shapes(ctx, kernel):
    from gpax_b200 import vExactGP
    X, y = dummy_data()
    Xt, _ = dummy_data(1)
    m = vExactGP(1, kernel, ctx=ctx)
    m.fit(0, X, y, num_warmup=50, num_samples=50, num_chains=2, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert s["k_length"].shape == (100, 3, 1) and s["k_scale"].shape == (100, 3) and s["noise"].shape == (100, 3)
    if kernel == "Periodic":
        assert s["period"].shape == (100, 3)
    sc = m.get_samples(chain_dim=True)
    assert sc["k_length"].shape == (2, 50, 3, 1) and sc["k_scale"].ndim == 3
    assert all(np.isfinite(v).all() for v in s.values())
    for n in (1, 10):
        mean, ys = m.predict(1, Xt[..., None], n=n)
        assert mean.shape == (3, 8) and ys.shape == (100, n, 3, 8)
        m1, y1 = m.predict_in_batches(1, Xt, batch_size=4, n=n, noiseless=True)
        m2, y2 = m.predict_in_batches(1, Xt, batch_size=4, n=n, noiseless=False)
        assert m1.shape == (3, 8) and y1.shape == (100, n, 3, 8)
        assert np.array_equal(m1, m2) and np.count_nonzero(y1 - y2) > 0
    one = {k: v[0] for k, v in s.items()}
    mean, cov = m.get_mvn_posterior(Xt[..., None], one)
    assert mean.shape == (3, 8) and cov.shape == (3, 8, 8)


def test_vexact_recovers_the_order_of_task_lengthscales(ctx):
    from gpax_b200 import vExactGP
    rng = np.random.default_rng(5)
    N = 40
    X = np.stack([np.sort(rng.uniform(0, 1, N)) for _ in range(2)])
    y = []
    for b, ell in enumerate((0.1, 1.0)):
        K = np.exp(-0.5 * (X[b][:, None] - X[b][None, :]) ** 2 / ell ** 2) + 1e-4 * np.eye(N)
        y.append(np.linalg.cholesky(K) @ rng.standard_normal(N) + 0.01 * rng.standard_normal(N))
    m = vExactGP(1, "RBF", ctx=ctx)
    m.fit(1, X, np.array(y), num_warmup=200, num_samples=200, progress_bar=False, print_summary=False)
    med = np.median(m.get_samples()["k_length"][:, :, 0], axis=0)
    assert med[0] < med[1], med


@pytest.mark.parametrize("sx_prior", [False, True])
def test_uigp_fit_predict(ctx, sx_prior):
    from gpax_b200 import UIGP
    from gpax_b200 import priors as P
    rng = np.random.default_rng(2)
    X = np.linspace(0, 1, 20)
    y = np.sin(6 * X) + 0.05 * rng.standard_normal(20)
    m = UIGP(1, "RBF", sigma_x_prior_dist=P.HalfNormal(0.05) if sx_prior else None, ctx=ctx)
    m.fit(0, X, y, num_warmup=50, num_samples=50, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert s["sigma_x"].shape == (50, 1) and s["X_prime"].shape == (50, 20, 1) and s["k_length"].shape == (50, 1)
    assert all(np.isfinite(v).all() for v in s.values())
    Xt = np.linspace(0, 1, 15)
    mean, ys = m.predict(1, Xt, n=2)
    assert mean.shape == (15,) and ys.shape == (50, 2, 15) and np.isfinite(ys).all()
    mu, cov = m.get_mvn_posterior(Xt[:, None], {k: v[0] for k, v in s.items()})
    assert mu.shape == (15,) and cov.shape == (15, 15)


def test_uigp_fit_at_300_points_takes_the_large_route(ctx):
    from gpax_b200 import UIGP
    rng = np.random.default_rng(3)
    X = rng.uniform(0, 1, 300)
    X[0], X[1] = 0.0, 1.0
    y = np.sin(6 * X) + 0.05 * rng.standard_normal(300)
    m = UIGP(1, "Matern", ctx=ctx)
    c0 = ctx.path_counts()["mll_batch_small"]
    m.fit(0, X, y, num_warmup=5, num_samples=5, progress_bar=False, print_summary=False)
    assert ctx.path_counts()["mll_batch_small"] == c0
    s = m.get_samples()
    assert s["X_prime"].shape == (5, 300, 1) and all(np.isfinite(v).all() for v in s.values())
