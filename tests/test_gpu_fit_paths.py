"""GPU: the fit-side entry points (b2gp_mll, b2gp_mll_v, b2gp_sparse_elbo, b2gp_mvn_sample) against closed-form references
(oracle/fit_oracle.py) on every solve route, each under options NAMED in the test and with the path counters it moved.

Tolerances, one rule for the whole file (fit_oracle.tau):
  value                   |v - ref| <= 1e-9 |ref|
  each gradient entry     |g - ref| <= tau (|ref| + scale), scale = the size of the terms that cancel in that entry
  tau on fp64 routes      1e-9 max(1, cond / 1e5), the parity bar of test_gpu_paths.py; cond = cond(K) or cond(Kuu)
  tau on int8 routes      INT8_SAFETY * cond * max(C_PLANES[S], 2^-53): DESIGN 4.6's digit-plane model, floored at fp64's
                          unit roundoff
tests/test_fit_oracle_cpu.py checks that the references agree with 60-digit arithmetic and that each named defect
(fit_oracle MUTATIONS) breaks the tolerance of the case here that stands for it.  Each test prints its largest err / tau
("err/tau <route> <case> <ratio>", visible with -s).  Nothing here touches gpax_b200.default_context()."""
import ctypes as C

import numpy as np
import pytest

from oracle import fit_oracle as fo

pytestmark = pytest.mark.gpu

JITTER = 1e-6


@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def counted(ctx, fn):
    """fn() and the path counters it moved"""
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


def report(route, case, ratio):
    print(f"err/tau {route} {case} {ratio:.3g}")
    assert ratio <= 1.0, (route, case, ratio)


def split_point(n):                      # potrf.cuh
    h = -(-((n + 1) // 2) // 128) * 128
    return n - (128 if n > 128 else 0) if h >= n else h


def trsm_panel_solves(m, n, panel):
    """panel solves of trsm_rec(m right-hand sides, n columns) with ozaki != 0"""
    if m < 1024 or n <= 128:
        return 0
    if n <= panel:
        return 1
    if n <= 256:                         # trsm_strip
        return 0
    n1 = split_point(n)
    return trsm_panel_solves(m, n1, panel) + trsm_panel_solves(m, n - n1, panel)


def tall_panel_solves(n, r, nb):
    """panel solves of potrf_tall(n, r rows below) with panel width nb"""
    if n <= nb:
        return 1 if r > 0 else 0
    n1 = (-(-n // nb) + 1) // 2 * nb
    return tall_panel_solves(n1, n - n1 + r, nb) + tall_panel_solves(n - n1, r, nb)


# ------------------------------------------------------------------ exact-GP likelihood
def check_mll(ctx, kind, X, y, theta, planes, route, noise_vec=None):
    """value, every gradient entry, alpha (and d/d noise_vec) against fit_oracle.mll_grad; returns the counters moved"""
    N = X.shape[0]
    v, g, a, gnv, sc = fo.mll_grad(kind, X, y, theta, JITTER, noise_vec)
    t = fo.tau(fo.mll_cond(kind, X, theta, JITTER, noise_vec), planes)
    out, c = counted(ctx, lambda: ctx.mll(kind, X, y, theta, JITTER, want_grad=True, want_alpha=True, noise_vec=noise_vec))
    val, grad, alpha, info = out[:4]
    case = f"{kind}-N{N}-d{X.shape[1]}"
    assert info == 0, case
    assert abs(val - v) <= 1e-9 * abs(v), (case, val, v)
    r = max(fo.err_ratio(grad, g, sc, t), fo.err_ratio(alpha, a, np.abs(a).max(), t))
    if noise_vec is not None:
        r = max(r, fo.err_ratio(out[4], gnv, a ** 2 - gnv, t))   # 1/2 (alpha^2 + diag K^-1)
    report(route, case, r)
    return c


DEFAULT_N = [1, 2, 7, 63, 64, 65, 129, 257, 1025, 2049]


def mll_default_case(N):
    """(kind, X, y, theta) of test_mll_default_options at N"""
    kind = ("RBF", "Matern", "Periodic")[DEFAULT_N.index(N) % 3]
    return (kind,) + fo.mll_problem(kind, N, 2, N)


@pytest.mark.parametrize("N", DEFAULT_N)
def test_mll_default_options(ctx, N):
    """the shipped options (ozaki = 0): every size is fp64, one 128-leaf factorisation per diagonal block"""
    kind, X, y, theta = mll_default_case(N)
    c = check_mll(ctx, kind, X, y, theta, 0, "fp64")
    assert c["potrf_diag"] == -(-N // 128) and c["oz_mma"] == c["potrf_tall"] == c["panel_solve"] == 0, c


@pytest.mark.parametrize("kind,N", [("Matern", 129), ("Periodic", 1025)])
def test_mll_d16(ctx, kind, N):
    """d = MLL_MAX_D, with 64-tiles that end ragged"""
    X, y, theta = fo.mll_problem(kind, N, 16, 16 + N)
    c = check_mll(ctx, kind, X, y, theta, 0, "fp64")
    assert c["oz_mma"] == 0, c


@pytest.mark.parametrize("ozaki", [7, 6])
@pytest.mark.parametrize("N,panel", [(300, 128), (1100, 256)])
def test_mll_tall_route(ctx, N, panel, ozaki):
    """potrf_tall from tall_min = 256: at N = 300 with 128-wide panels the last one is 44 rows; at N = 1100 with 256-wide
    panels trsm_rec also solves B^T = L^-T (N rows >= 1024) by the panel route, which needs 128 < block <= panel"""
    kind = "Matern" if N == 300 else "RBF"
    X, y, theta = fo.mll_problem(kind, N, 3, N + ozaki)
    with ctx.options(ozaki=ozaki, tall_min=256, panel=panel):
        c = check_mll(ctx, kind, X, y, theta, ozaki, f"int8-{ozaki}-tall-panel{panel}")
    solves = tall_panel_solves(N, 1, panel) + trsm_panel_solves(N, N, panel)
    assert c["potrf_tall"] == 1 and c["panel_solve"] == solves and c["oz_mma"] >= solves, c
    if N == 1100:
        assert trsm_panel_solves(N, N, panel) > 0


def kinv_syrk_case():
    return fo.mll_problem("RBF", 600, 1, 600, noise=1.0, ell=0.01)


def test_mll_kinv_syrk_on_int8(ctx):
    """K^-1 = L^-T L^-1 is the one product of an N = 600 likelihood that qualifies for the int8 path (k = N >= 512, 30
    lower 128 x 64 tiles): with oz_min_tiles = 30 it runs there, and nothing else does"""
    X, y, theta = kinv_syrk_case()
    with ctx.options(ozaki=7, oz_min_tiles=30):
        c = check_mll(ctx, "RBF", X, y, theta, 7, "int8-7-kinv-syrk")
    assert c["oz_mma"] == 1 and c["potrf_tall"] == c["panel_solve"] == 0, c


def test_mll_ozaki7_default_options(ctx):
    """N = 2049 >= tall_min with the shipped panel width: tall factorisation, panel-route B^T solve, int8 SYRK"""
    X, y, theta = fo.mll_problem("Matern", 2049, 2, 4049)
    with ctx.options(ozaki=7):
        c = check_mll(ctx, "Matern", X, y, theta, 7, "int8-7-default")
    solves = tall_panel_solves(2049, 1, 1024) + trsm_panel_solves(2049, 2049, 1024)
    assert c["potrf_tall"] == 1 and c["panel_solve"] == solves and c["oz_mma"] > solves, c


@pytest.mark.parametrize("N,ozaki", [(65, 0), (1025, 0), (2049, 7)])
def test_mll_v_noise_vec(ctx, N, ozaki):
    """per-point noise variances over 1e-4 .. 1 on the diagonal and d value / d noise_vec"""
    X, y, theta = fo.mll_problem("RBF", N, 2, N + 7, noise=1e-3)
    nv = np.random.default_rng(N).permutation(np.geomspace(1e-4, 1.0, N))
    with ctx.options(ozaki=ozaki):
        c = check_mll(ctx, "RBF", X, y, theta, ozaki, "int8-7-default" if ozaki else "fp64", noise_vec=nv)
    assert (c["potrf_tall"] == 1) == (ozaki != 0), c


# ------------------------------------------------------------------ VFE bound
def check_elbo(ctx, kind, Xu, X, y, theta, planes, route, jitter=1e-5):
    v, g, gx, sc, sx, T = fo.elbo_grad(kind, Xu, X, y, theta, jitter)
    t = fo.tau(fo.kuu_cond(kind, Xu, theta, jitter), planes)
    (val, grad, gxu, info), c = counted(ctx, lambda: ctx.sparse_elbo(kind, Xu, X, y, theta, jitter))
    case = f"{kind}-M{Xu.shape[0]}-N{X.shape[0]}-d{X.shape[1]}-T{'+' if T > 0 else '-'}"
    assert info == 0, case
    assert abs(val - v) <= 1e-9 * abs(v), (case, val, v)
    report(route, case, max(fo.err_ratio(grad, g, sc, t), fo.err_ratio(gxu, gx, sx, t)))   # all M x d entries of grad_Xu
    return c, T


ELBO_SHAPES = [(1, 50, 1), (7, 61, 16), (128, 1000, 3), (129, 1001, 3), (257, 700, 1), (50, 30, 16), (300, 300, 3)]


def elbo_default_case(M, N, d):
    """(kind, Xu, X, y, theta) of test_elbo_default_options"""
    kind = ("RBF", "Matern", "Periodic")[ELBO_SHAPES.index((M, N, d)) % 3]
    return (kind,) + fo.elbo_problem(kind, M, N, d, M + N, xu_is_x=(M == N))


@pytest.mark.parametrize("M,N,d", ELBO_SHAPES)
def test_elbo_default_options(ctx, M, N, d):
    """one 128-leaf (M <= 128), the recursion just past it, N < M, and Xu = X (Kuu = Kff + jitter I)"""
    kind, Xu, X, y, theta = elbo_default_case(M, N, d)
    (c, T) = check_elbo(ctx, kind, Xu, X, y, theta, 0, "fp64")
    assert T > 0 and c["oz_mma"] == c["potrf_tall"] == c["panel_solve"] == 0, c


def test_elbo_tall_panel_int8_route(ctx):
    """M = 300, N = 1100 under ozaki = 7, tall_min = 256, panel = 256, oz_min_tiles = 12: potrf_tall on Kuu (a 256 block and
    a ragged 44-row block), the panel route for W^T = Kfu Luu^-T (1100 rows), the int8 W W^T (3 x 4 lower tiles)"""
    M, N = 300, 1100
    Xu, X, y, theta = fo.elbo_problem("Matern", M, N, 2, 11)
    with ctx.options(ozaki=7, tall_min=256, panel=256, oz_min_tiles=12):
        c, _ = check_elbo(ctx, "Matern", Xu, X, y, theta, 7, "int8-7-elbo-tall")
    solves = tall_panel_solves(M, 0, 256) + trsm_panel_solves(N, M, 256)
    assert c["potrf_tall"] == 1 and c["panel_solve"] == solves and c["oz_mma"] == solves + 1, c


def test_elbo_large_m_panel_route(ctx):
    """M = 1100 at ozaki = 7: BtC = LC^-T and BtU = Luu^-T (M rows each) and W^T take the panel route"""
    M, N = 1100, 1200
    Xu, X, y, theta = fo.elbo_problem("RBF", M, N, 3, 12)
    theta[:3] = 0.12
    with ctx.options(ozaki=7):
        c, _ = check_elbo(ctx, "RBF", Xu, X, y, theta, 7, "int8-7-elbo-panel")
    solves = 2 * trsm_panel_solves(M, M, 1024) + trsm_panel_solves(N, M, 1024)
    assert c["potrf_tall"] == 0 and c["panel_solve"] == solves and solves >= 6, c


def separated_problem(kind, n, d=1):
    """points 5 lengthscales apart: Kff is the identity times k_scale up to 4e-6"""
    rng = np.random.default_rng(n)
    X = np.arange(n, dtype=float)[:, None] * 0.5 + np.zeros((1, d))
    y = rng.standard_normal(n)
    theta = np.concatenate([np.full(d, 0.1), [1.3, 0.2, 1.0]])
    return X, y, theta


@pytest.mark.parametrize("kind", ["RBF", "Matern"])
def test_elbo_both_sides_of_the_clip(ctx, kind):
    """Xu = X, points far apart: jitter > 0 gives T > 0 (the trace term counts); jitter = -1e-4 makes Q_nn > K_nn exactly,
    T < 0, and the clip zeroes the term and its gradient (coef = 0 in elbo_gw_kernel, no host corrections)"""
    X, y, theta = separated_problem(kind, 40)
    for jitter, sign in ((1e-5, 1), (-1e-4, -1)):
        c, T = check_elbo(ctx, kind, X, X, y, theta, 0, "fp64", jitter=jitter)
        assert np.sign(T) == sign and abs(T) > 1e-3 * abs(jitter) * 40, (jitter, T)


# ------------------------------------------------------------------ sampling from a covariance
def mvn_problem(S, P, n, seed):
    rng = np.random.default_rng(seed)
    mean = rng.standard_normal((S, P))
    covs = []
    for _ in range(S):
        G = rng.standard_normal((P, P)) / np.sqrt(P)
        covs.append(G @ G.T + 0.05 * np.eye(P))
    return mean, np.stack(covs), rng.standard_normal((S, n, P))


@pytest.mark.parametrize("ozaki", [0, 7])
@pytest.mark.parametrize("n", [1, 5])
@pytest.mark.parametrize("P", [1, 129, 1025, 2100])
def test_mvn_sample(ctx, P, n, ozaki):
    """y = mean + eps chol(cov)^T per member; with oz_min_tiles = 16 the trailing updates of P >= 1025 take the int8 path
    under ozaki = 7"""
    S = 3
    mean, cov, eps = mvn_problem(S, P, n, P + n)
    with ctx.options(ozaki=ozaki, oz_min_tiles=16):
        (y, info), c = counted(ctx, lambda: ctx.mvn_sample(mean, cov, eps))
    assert (info == 0).all()
    planes = 7 if c["oz_mma"] else 0
    assert (c["oz_mma"] > 0) == (ozaki == 7 and P >= 1025), c
    r = 0.0
    for s in range(S):
        L = np.linalg.cholesky(cov[s])
        ev = np.linalg.eigvalsh(cov[s])
        ref = mean[s] + eps[s] @ L.T
        r = max(r, fo.err_ratio(y[s], ref, np.abs(eps[s]) @ np.abs(L).T, fo.tau(ev[-1] / ev[0], planes)))
    report("int8-7-mvn" if planes else "fp64", f"mvn-P{P}-n{n}", r)


def test_mvn_sample_bad_member(ctx):
    """one member not positive definite: info > 0 and NaN rows there, the other members bit-identical to a call where
    every member is positive definite"""
    mean, cov, eps = mvn_problem(3, 300, 4, 1)
    bad = cov.copy()
    bad[1, 7, 7] = -1.0
    good, info0 = ctx.mvn_sample(mean, cov, eps)
    y, info = ctx.mvn_sample(mean, bad, eps)
    assert (info0 == 0).all() and info[1] > 0 and info[0] == info[2] == 0, info
    assert np.isnan(y[1]).all()
    np.testing.assert_array_equal(y[[0, 2]], good[[0, 2]])


# ------------------------------------------------------------------ invariants
def fit_calls(ctx):
    """one call of every fit entry point on an int8-eligible size: name -> callable returning a tuple of arrays"""
    X, y, theta = fo.mll_problem("Matern", 2049, 2, 5)
    nv = np.geomspace(1e-4, 1.0, 2049)
    Xu, Xs, ys, ths = fo.elbo_problem("RBF", 300, 1100, 2, 6)
    mean, cov, eps = mvn_problem(2, 2100, 2, 3)

    def as_arrays(t):
        return tuple(np.atleast_1d(np.asarray(v, dtype=float)) for v in t if v is not None)
    return {
        "mll": lambda: as_arrays(ctx.mll("Matern", X, y, theta, JITTER, want_grad=True, want_alpha=True)),
        "mll_v": lambda: as_arrays(ctx.mll("Matern", X, y, theta, JITTER, want_grad=True, want_alpha=True, noise_vec=nv)),
        "sparse_elbo": lambda: as_arrays(ctx.sparse_elbo("RBF", Xu, Xs, ys, ths, 1e-5)),
        "mvn_sample": lambda: as_arrays(ctx.mvn_sample(mean, cov, eps)),
    }


def test_identical_calls_identical_bits_and_auto_ozaki_is_seven_planes(ctx):
    """fixed-order reductions: the same call gives the same bits; outside the posterior ozaki = -1 takes 7 digit planes,
    so it is bit-identical to ozaki = 7 (and uses the int8 path at these sizes)"""
    for name, fn in fit_calls(ctx).items():
        with ctx.options(ozaki=7, tall_min=2048 if name != "sparse_elbo" else 256, panel=1024 if name != "sparse_elbo" else 256,
                         oz_min_tiles=12):
            a, c = counted(ctx, fn)
            b = fn()
            ctx.set_option("ozaki", -1)
            m = fn()
        assert c["oz_mma"] > 0, (name, c)
        for u, v, w in zip(a, b, m):
            np.testing.assert_array_equal(u, v, err_msg=f"{name}: repeated call")
            np.testing.assert_array_equal(u, w, err_msg=f"{name}: ozaki -1 against 7")


def test_mll_value_bits_do_not_depend_on_what_else_is_requested(ctx):
    X, y, theta = fo.mll_problem("Periodic", 1025, 2, 9)
    for ozaki in (0, 7):
        with ctx.options(ozaki=ozaki, tall_min=256):
            full = ctx.mll("Periodic", X, y, theta, JITTER, want_grad=True, want_alpha=True)
            bare = ctx.mll("Periodic", X, y, theta, JITTER, want_grad=False, want_alpha=False)
            only_alpha = ctx.mll("Periodic", X, y, theta, JITTER, want_grad=False, want_alpha=True)
        assert full[0] == bare[0] == only_alpha[0], ozaki
        np.testing.assert_array_equal(full[2], only_alpha[2])


def test_device_pointer_inputs_match_host_inputs(ctx):
    """B2GP_FLAG_DEVICE_PTRS: X, y (and Xu) already on the device give the bits of the host-array call"""
    from gpax_b200 import _ffi
    lib = ctx.lib
    X, y, theta = fo.mll_problem("RBF", 700, 3, 21)
    N, d = X.shape
    v0, g0, _, _ = ctx.mll("RBF", X, y, theta, JITTER)
    dX, dy = ctx.to_device(X), ctx.to_device(y)
    val, info, g = C.c_double(), C.c_int(), np.zeros(d + 3)
    ctx._check(lib.b2gp_mll(ctx.h, _ffi.KERNEL_RBF, dX.ptr, N, dy.ptr, d, _ffi._ptr(theta), JITTER, _ffi.FLAG_DEVICE_PTRS,
                            C.byref(val), _ffi._ptr(g), None, C.byref(info)))
    assert info.value == 0 and val.value == v0
    np.testing.assert_array_equal(g, g0)
    Xu, Xs, ys, ths = fo.elbo_problem("Matern", 150, 600, 2, 22)
    e0, eg0, ex0, _ = ctx.sparse_elbo("Matern", Xu, Xs, ys, ths, 1e-5)
    dXu, dXs, dys = ctx.to_device(Xu), ctx.to_device(Xs), ctx.to_device(ys)
    g, gx = np.zeros(5), np.zeros((150, 2))
    ctx._check(lib.b2gp_sparse_elbo(ctx.h, _ffi.KERNEL_MATERN52, dXu.ptr, 150, dXs.ptr, 600, dys.ptr, 2, _ffi._ptr(ths), 1e-5,
                                    _ffi.FLAG_DEVICE_PTRS, C.byref(val), _ffi._ptr(g), _ffi._ptr(gx), C.byref(info)))
    assert info.value == 0 and val.value == e0
    np.testing.assert_array_equal(g, eg0)
    np.testing.assert_array_equal(gx, ex0)


@pytest.mark.parametrize("fit", ["mll", "sparse_elbo"])
def test_fit_calls_invalidate_the_factor_cache(ctx, fit):
    """b2gp_mll and b2gp_sparse_elbo overwrite slot 0's matrix: the next posterior with the same theta factors again (no
    cache hit) and gives the bits of the first one"""
    X, y, theta = fo.mll_problem("Matern", 800, 2, 31)
    Xn = np.random.default_rng(32).uniform(0, 1, (60, 2))
    first = ctx.posterior("Matern", X, y, Xn, theta[None], want=("mean", "var", "cov"))
    hits = ctx.cache_hits()
    if fit == "mll":
        ctx.mll("Matern", X, y, theta, JITTER, want_grad=True, want_alpha=True)
    else:
        ctx.sparse_elbo("Matern", X[:700], X, y, theta, 1e-5)
    again = ctx.posterior("Matern", X, y, Xn, theta[None], want=("mean", "var", "cov"))
    assert ctx.cache_hits() == hits
    for k in ("mean", "var", "cov"):
        np.testing.assert_array_equal(again[k], first[k], err_msg=k)


def test_mvn_sample_keeps_the_factor_cache(ctx):
    """b2gp_mvn_sample works in slot 0's covariance scratch only: after P = 2100 on the int8 path the same posterior is
    still a cache hit, with the bits of the cache hit before it.  (A hit is compared with a hit: at N >= tall_min the
    factoring call solves k_pX inside the tall factorisation's panel solves and a hit solves it by trsm_tall, so the two
    agree within the digit-plane error, not bit for bit.)"""
    X, y, theta = fo.mll_problem("RBF", 2500, 2, 41)
    Xn = np.random.default_rng(42).uniform(0, 1, (80, 2))
    mean, cov, eps = mvn_problem(1, 2100, 2, 43)
    with ctx.options(ozaki=7, oz_min_tiles=16):
        ctx.posterior("RBF", X, y, Xn, theta[None], want=("mean", "var", "cov"))
        first = ctx.posterior("RBF", X, y, Xn, theta[None], want=("mean", "var", "cov"))
        hits = ctx.cache_hits()
        (_, info), c = counted(ctx, lambda: ctx.mvn_sample(mean, cov, eps))
        assert (info == 0).all() and c["oz_mma"] > 0, c
        again = ctx.posterior("RBF", X, y, Xn, theta[None], want=("mean", "var", "cov"))
    assert hits >= 1 and ctx.cache_hits() == hits + 1
    for k in ("mean", "var", "cov"):
        np.testing.assert_array_equal(again[k], first[k], err_msg=k)


# ------------------------------------------------------------------ failures
def test_mll_not_positive_definite_on_the_tall_route(ctx):
    X, y, theta = fo.mll_problem("RBF", 300, 2, 51)
    theta[2] = -1.0                                          # k_scale < 0
    with ctx.options(ozaki=7, tall_min=256, panel=128):
        (val, grad, alpha, info, gnv), c = counted(ctx, lambda: ctx.mll("RBF", X, y, theta, JITTER, noise_vec=np.full(300, 1e-3)))
    assert c["potrf_tall"] == 1, c
    assert info > 0 and np.isnan(val) and np.isnan(grad).all() and np.isnan(gnv).all()


def test_elbo_not_positive_definite_kuu_gives_nan_everywhere(ctx):
    """a failed Kuu factorisation: info > 0 and NaN in the value, grad_theta and grad_Xu.  grad_Xu is set to NaN on the
    host like the other outputs, so the contract does not rest on NaN propagating through the reverse pass"""
    Xu, X, y, theta = fo.elbo_problem("RBF", 40, 200, 2, 61)
    theta[2] = -1.0
    val, g, gx, info = ctx.sparse_elbo("RBF", Xu, X, y, theta, 1e-5)
    assert info > 0 and np.isnan(val) and np.isnan(g).all() and np.isnan(gx).all(), (info, gx[:2])


def test_d17_is_refused(ctx):
    from gpax_b200 import _ffi
    d = 17
    X, y, th = np.random.default_rng(0).uniform(0, 1, (20, d)), np.ones(20), np.ones(d + 3)
    val, info, g, gx = C.c_double(), C.c_int(), np.zeros(d + 3), np.zeros((4, d))
    rc = ctx.lib.b2gp_mll(ctx.h, 0, _ffi._ptr(X), 20, _ffi._ptr(y), d, _ffi._ptr(th), JITTER, 0, C.byref(val), _ffi._ptr(g), None,
                          C.byref(info))
    assert rc == -1                                          # B2GP_ERR_ARG
    rc = ctx.lib.b2gp_mll_v(ctx.h, 0, _ffi._ptr(X), 20, _ffi._ptr(y), d, _ffi._ptr(th), _ffi._ptr(y), JITTER, 0, C.byref(val),
                            _ffi._ptr(g), None, _ffi._ptr(np.zeros(20)), C.byref(info))
    assert rc == -1
    rc = ctx.lib.b2gp_sparse_elbo(ctx.h, 0, _ffi._ptr(X[:4].copy()), 4, _ffi._ptr(X), 20, _ffi._ptr(y), d, _ffi._ptr(th), JITTER, 0,
                                  C.byref(val), _ffi._ptr(g), _ffi._ptr(gx), C.byref(info))
    assert rc == -1
