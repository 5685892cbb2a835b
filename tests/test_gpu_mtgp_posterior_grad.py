"""GPU: the LCM posterior's gradient w.r.t. the test inputs (b2gp_posterior_multitask_grad, gram_dx_lcm_kernel) and
optimize_acq on MultiTaskGP / CoregGP built on it.

dmean / dvar are held to tests/mtgp_grad_oracle.py (pinned on the CPU by central differences of
oracle/mtgp_oracle.posterior) at 1e-9, scaled by cond(K) / 1e5 above cond(K) = 1e5, as test_gpu_posterior_grad.py does.
mean and var are b2gp_posterior_multitask's bit for bit under ozaki 0 on the recursive route, the fp64 tall-panel route
and its lock-step draw groups."""
import itertools

import numpy as np
import pytest

from conftest import assert_close
from mtgp_grad_oracle import posterior_grad as oracle_grad
from oracle import mtgp_oracle as mo

pytestmark = pytest.mark.gpu

RTOL = 1e-9
ALL = ("mean", "var", "dmean", "dvar")


@pytest.fixture(scope="module")
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def counted(ctx, fn):
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


def params(rng, L, T, d, kind, S):
    return {"k_length": rng.uniform(0.4, 0.9, (S, L, d)) * np.sqrt(d), "k_scale": rng.uniform(0.8, 1.3, (S, L)),
            "W": rng.normal(0, 0.7, (S, L, T, 2)), "v": rng.uniform(0.3, 0.8, (S, L, T)), "noise": rng.uniform(0.05, 0.2, (S, T)),
            "period": rng.uniform(1.5, 2.5, (S, L)) if kind == "Periodic" else None}


def draw(p, s):
    return {k: (None if v is None else np.asarray(v)[s]) for k, v in p.items()}


def packed(p, T, d):
    S, L = p["k_scale"].shape
    th = np.empty((S, L, d + 2))
    th[..., :d] = p["k_length"]
    th[..., d] = p["k_scale"]
    th[..., d + 1] = 1.0 if p["period"] is None else p["period"]
    B = np.einsum("sltr,slur->sltu", p["W"], p["W"]) + p["v"][..., None] * np.eye(T)
    return th, B, p["noise"]


def problem(kind, L, T, d, S, P, shared, n_rows, seed=0):
    """inputs with task columns (multitask form) or points (Kronecker form, n_rows // T of them), P test points"""
    rng = np.random.default_rng(seed + 1000 * L + 100 * T + 10 * d + S + 7 * P + shared)
    n = n_rows // T if shared else n_rows
    X = rng.uniform(0, 2, (n, d))
    Xn = rng.uniform(0, 2, (P, d))
    if not shared:
        X = np.c_[X, np.arange(n) % T]
        Xn = np.c_[Xn, rng.integers(0, T, P)]
    y = rng.standard_normal(n * T if shared else n)
    return X, y, Xn, params(rng, L, T, d, kind, S)


def call(ctx, kind, X, y, Xn, p, T, d, shared, grad=True, noiseless=False, want=None):
    Xd, tt, g = mo.expand(X, shared, T)
    Xnd, tn, _ = mo.expand(Xn, shared, T)
    th, B, nz = packed(p, T, d)
    if grad:
        return ctx.posterior_multitask_grad(kind, Xd, tt, y, Xnd, tn, th, B, nz, g, noiseless, 1e-6, want or ALL)
    return ctx.posterior_multitask(kind, Xd, tt, y, Xnd, tn, th, B, nz, g, noiseless, 1e-6, want or ("mean", "var"))


def check_oracle(out, kind, X, y, Xn, p, T, shared, noiseless, what):
    for s in range(len(out["info"])):
        ps = draw(p, s)
        assert out["info"][s] == 0, what
        K = mo.lcm_cov(X, X, ps, np.asarray(ps["noise"]), kind, shared, T)
        cond = np.linalg.cond(K)
        tol = RTOL * max(1.0, cond / 1e5)
        ref = oracle_grad(X, y, Xn, ps, kind, shared, T, noiseless)
        for name, r in zip(ALL, ref):
            r = r if shared or r.ndim == 1 else r[:, :-1]          # the library returns the data columns only
            assert_close(out[name][s], r, tol, f"{name} draw {s} {what}, cond(K) = {cond:.3g}")


ORACLE_CASES = list(itertools.product(["RBF", "Matern", "Periodic"], [1, 4], [2, 8], [1, 3, 16], [False, True]))


@pytest.mark.parametrize("kind,L,T,d,shared", ORACLE_CASES)
def test_gradient_vs_oracle(ctx, kind, L, T, d, shared):
    for S, P in ((1, 1), (4, 17)):
        noiseless = (S == 4)
        X, y, Xn, p = problem(kind, L, T, d, S, P, shared, 64)
        with ctx.options(ozaki=0):
            out = call(ctx, kind, X, y, Xn, p, T, d, shared, noiseless=noiseless)
        assert out["dmean"].shape == (S, P * (T if shared else 1), d)
        check_oracle(out, kind, X, y, Xn, p, T, shared, noiseless, f"{kind} L={L} T={T} d={d} S={S} P={P} shared={shared}")


def same_as_plain(ctx, kind, X, y, Xn, p, T, d, shared, what, **opts):
    with ctx.options(**opts):
        out, moved = counted(ctx, lambda: call(ctx, kind, X, y, Xn, p, T, d, shared))
        plain, moved_plain = counted(ctx, lambda: call(ctx, kind, X, y, Xn, p, T, d, shared, grad=False))
    for name in ("mean", "var"):
        assert np.array_equal(out[name], plain[name]), f"{name} {what}"
    return out, moved, moved_plain


@pytest.mark.parametrize("kind,shared", [("RBF", False), ("Matern", True), ("Periodic", False)])
def test_mean_var_bit_identical_recursive_route(ctx, kind, shared):
    X, y, Xn, p = problem(kind, 2, 3, 3, 2, 17, shared, 300)
    out, moved, _ = same_as_plain(ctx, kind, X, y, Xn, p, 3, 3, shared, f"{kind} recursive", ozaki=0)
    assert moved["potrf_tall_fp64"] == 0 and moved["potrf_diag"] > 0, moved
    check_oracle(out, kind, X, y, Xn, p, 3, shared, False, f"{kind} recursive")


@pytest.mark.parametrize("kind,shared", [("Matern", False), ("RBF", True)])
def test_mean_var_bit_identical_tall_fp64_route(ctx, kind, shared):
    X, y, Xn, p = problem(kind, 2, 2, 3, 1, 9, shared, 640)
    out, moved, moved_plain = same_as_plain(ctx, kind, X, y, Xn, p, 2, 3, shared, f"{kind} tall fp64", ozaki=0, tall_min_fp64=256,
                                                panel=256)
    assert moved["potrf_tall_fp64"] == 1 and moved_plain["potrf_tall_fp64"] == 1, moved
    check_oracle(out, kind, X, y, Xn, p, 2, shared, False, f"{kind} tall fp64")


def test_mean_var_bit_identical_lock_step_draw_groups(ctx):
    S = 8
    X, y, Xn, p = problem("Matern", 2, 3, 2, S, 5, False, 640)
    out, moved, moved_plain = same_as_plain(ctx, "Matern", X, y, Xn, p, 3, 2, False, "lock-step groups", ozaki=0,
                                            tall_min_fp64=256, panel=256, streams=8)
    assert moved["potrf_tall_batch"] == 2 and moved_plain["potrf_tall_batch"] == 2, moved     # two groups of 4
    check_oracle(out, "Matern", X, y, Xn, p, 3, False, False, "lock-step groups")


def test_int8_route_meets_the_oracle(ctx):
    """ozaki 7 on the int8 tall-panel route: the extra rows may cross an int8 dispatch threshold, so the oracle only"""
    X, y, Xn, p = problem("RBF", 2, 2, 2, 2, 20, False, 2500)
    with ctx.options(ozaki=7):
        out, moved = counted(ctx, lambda: call(ctx, "RBF", X, y, Xn, p, 2, 2, False))
    assert moved["potrf_tall"] == 2, moved
    check_oracle(out, "RBF", X, y, Xn, p, 2, False, False, "int8 tall route")


def test_outputs_subset_and_mean_only(ctx):
    X, y, Xn, p = problem("RBF", 2, 2, 2, 2, 6, False, 100)
    full = call(ctx, "RBF", X, y, Xn, p, 2, 2, False)
    part = call(ctx, "RBF", X, y, Xn, p, 2, 2, False, want=("dmean",))
    assert part["mean"] is None and part["var"] is None and part["dvar"] is None
    assert np.array_equal(part["dmean"], full["dmean"])


def test_failed_draw_is_nan_alone_and_calls_are_deterministic(ctx):
    X, y, Xn, p = problem("Matern", 2, 3, 2, 3, 7, False, 120)
    p["noise"][1] = -5.0                                     # k_XX of draw 1 is not positive definite
    out = call(ctx, "Matern", X, y, Xn, p, 3, 2, False)
    assert out["info"][1] > 0 and out["info"][0] == 0 and out["info"][2] == 0
    for name in ALL:
        assert np.isnan(out[name][1]).all(), name
        assert np.isfinite(out[name][[0, 2]]).all(), name
    again = call(ctx, "Matern", X, y, Xn, p, 3, 2, False)
    for name in ALL:
        assert np.array_equal(out[name], again[name], equal_nan=True), name
    good = {k: (None if v is None else v[[0, 2]]) for k, v in p.items()}
    check_oracle({k: (v[[0, 2]]) for k, v in out.items()}, "Matern", X, y, Xn, good, 3, False, False, "failed-draw neighbours")


def test_refusals_launch_nothing(ctx):
    import ctypes as C

    from gpax_b200 import _ffi
    rng = np.random.default_rng(6)

    def raw(kind=0, T=2, L=1, d=2, task=None, flags=0):
        X = rng.uniform(0, 1, (20, d))
        t = (np.arange(20) % T if task is None else task).astype(np.int32)
        th, B, nz = np.ones((1, L, d + 2)), np.tile(np.eye(T), (1, L, 1, 1)), np.full((1, T), 0.1)
        out = np.empty(4 * d)
        info = np.zeros(1, dtype=np.int32)
        return ctx.lib.b2gp_posterior_multitask_grad(
            ctx.h, kind, _ffi._ptr(X), _ffi._ptr(t), 20, _ffi._ptr(np.ones(20)), 0, _ffi._ptr(X[:4]), _ffi._ptr(t[:4]), 4, d, 1, T,
            L, 1, _ffi._ptr(th), _ffi._ptr(B), _ffi._ptr(nz), 0, 1e-6, flags | _ffi.OUT_DMEAN, None, None, _ffi._ptr(out), None,
            info.ctypes.data_as(C.c_void_p), None)

    assert raw() == 0
    cases = [({"flags": f}, -4) for f in (_ffi.FLAG_F32, _ffi.FLAG_DEVICE_PTRS, _ffi.OUT_COV, _ffi.OUT_SAMPLE)]
    cases += [({"kind": 3}, -1), ({"kind": 4}, -1), ({"T": 9}, -1), ({"L": 5}, -1), ({"d": 17}, -1),
              ({"task": np.r_[np.zeros(19, int), 2]}, -1), ({"task": np.r_[np.zeros(19, int), -1]}, -1)]
    for kw, code in cases:
        launches, paths = ctx.last_timing()["launches"], ctx.path_counts()
        assert raw(**kw) == code, kw
        assert ctx.last_timing()["launches"] == launches and ctx.path_counts() == paths, kw


def test_only_the_gradient_call_launches_the_derivative_rows(ctx):
    """Counted launches (b2gp_timing::launches, which test_gpu_launch_accounting.py holds to the CUDA profiler's count):
    the plain multi-task posterior queues the same launches with the gradient bits set (they are masked off), and the
    gradient call adds exactly gram_dx_lcm_kernel and rowdot_grad_kernel, one each per draw.  On the recursive route at
    this size every other launch covers all right-hand-side rows at once, so the P*d extra rows add no launch there."""
    from gpax_b200 import _ffi
    S = 2
    X, y, Xn, p = problem("RBF", 2, 2, 3, S, 5, False, 200)
    Xd, tt, g = mo.expand(X, False, 2)
    Xnd, tn, _ = mo.expand(Xn, False, 2)
    th, B, nz = packed(p, 2, 3)
    launches = lambda: ctx.last_timing()["launches"]     # noqa: E731
    with ctx.options(ozaki=0):
        plain = ctx.posterior_multitask("RBF", Xd, tt, y, Xnd, tn, th, B, nz, g, want=("mean", "var"))
        n_plain = launches()
        masked = ctx.posterior_multitask("RBF", Xd, tt, y, Xnd, tn, th, B, nz, g, want=("mean", "var"),
                                         flags=_ffi.OUT_DMEAN | _ffi.OUT_DVAR)
        n_masked = launches()
        grad = call(ctx, "RBF", X, y, Xn, p, 2, 3, False)
        n_grad = launches()
    assert n_plain > 0 and n_masked == n_plain, (n_plain, n_masked)
    assert n_grad == n_plain + 2 * S, (n_plain, n_grad)
    for name in ("mean", "var"):
        assert np.array_equal(masked[name], plain[name]) and np.array_equal(grad[name], plain[name]), name


# ------------------------------------------------------------------ optimize_acq on MultiTaskGP / CoregGP
class FakeMCMC:
    def __init__(self, samples):
        self.samples = samples

    def get_samples(self, group_by_chain=False):
        return self.samples


def bo_data(d=2, T=2, n=16, seed=21):
    rng = np.random.default_rng(seed)
    Xd = rng.uniform(-2, 2, (n, d))
    t = np.arange(n) % T
    y = (Xd ** 3).sum(1) - Xd.prod(1) + 0.5 * t
    return np.c_[Xd, t], y


def lcm_models(ctx, d=2, S=3):
    from gpax_b200 import CoregGP, MultiTaskGP
    X, y = bo_data(d)
    rng = np.random.default_rng(5)
    mt = MultiTaskGP(d, "RBF", num_latents=2, num_tasks=2, ctx=ctx)
    mt.X_train, mt.y_train = X, y
    mt.mcmc = FakeMCMC({"k_length": rng.uniform(1.0, 2.0, (S, 2, d)), "k_scale": rng.uniform(5, 10, (S, 2)),
                        "W": rng.normal(0, 0.7, (S, 2, 2, 1)), "v": rng.uniform(0.3, 0.8, (S, 2, 2)),
                        "noise": rng.uniform(0.001, 0.01, (S, 2))})
    cg = CoregGP(d, "Matern", ctx=ctx)
    cg.X_train, cg.y_train = X, y
    cg.mcmc = FakeMCMC({"k_length": rng.uniform(1.0, 2.0, (S, d)), "W": rng.normal(0, 2.0, (S, 2, 1)),
                        "v": rng.uniform(3.0, 8.0, (S, 2)), "noise": rng.uniform(0.001, 0.01, (S, 2))})
    return {"MultiTaskGP": mt, "CoregGP": cg}


def run_and_check(ctx, model, acq_name, monkeypatch, task=1.0):
    from gpax_b200 import acquisition as acq, prng
    d = model.kernel_dim + 1
    acq_fn = getattr(acq, acq_name)
    key = prng.PRNGKey(5)
    lb, ub = [-2.0] * (d - 1) + [task], [2.0] * (d - 1) + [task]
    kw = {"noiseless": True}
    assert acq._analytic_kind(acq_fn, model, kw) == acq_name

    calls = {"posterior_multitask": 0, "posterior_multitask_grad": 0, "evals": 0}
    for name in ("posterior_multitask", "posterior_multitask_grad"):
        fn = getattr(ctx, name)

        def wrapped(*a, _fn=fn, _name=name, **k):
            calls[_name] += 1
            return _fn(*a, **k)
        monkeypatch.setattr(ctx, name, wrapped)
    objective = acq._analytic_objective

    def counting_objective(*a, **k):
        f = objective(*a, **k)

        def g(x):
            calls["evals"] += 1
            return f(x)
        return g
    monkeypatch.setattr(acq, "_analytic_objective", counting_objective)
    x = acq.optimize_acq(key, model, acq_fn, 5, lb, ub, **kw)
    monkeypatch.setattr(acq, "_analytic_objective", objective)
    assert calls["evals"] >= 1 and calls["posterior_multitask_grad"] == calls["evals"], calls
    assert calls["posterior_multitask"] == 1, calls                       # the initial guesses' one predict
    assert x.shape == (d,) and np.all(x >= np.asarray(lb)) and np.all(x <= np.asarray(ub))
    guesses = prng.uniform(key, (5, d), np.float32, np.asarray(lb, np.float32), np.asarray(ub, np.float32))
    best0 = np.max(acq_fn(key, model, guesses, **kw))
    assert acq_fn(key, model, np.asarray(x, np.float64)[None], **kw)[0] >= best0 - 1e-12 * abs(best0)

    # value against acq_fn, gradient against its central differences on the free columns, 0 on the task column
    f = acq._analytic_objective(acq_name, key, model, d, kw)
    x0 = np.r_[np.linspace(-0.7, 0.4, d - 1), task]
    val, grad = f(x0)
    assert np.isclose(val, acq_fn(key, model, x0[None], **kw)[0], rtol=1e-12, atol=0), "value of the gradient path"
    assert grad[-1] == 0.0
    h, fd = 1e-5, np.empty(d - 1)
    for k in range(d - 1):
        e = np.zeros(d)
        e[k] = h
        fd[k] = (acq_fn(key, model, (x0 + e)[None], **kw)[0] - acq_fn(key, model, (x0 - e)[None], **kw)[0]) / (2 * h)
    np.testing.assert_allclose(grad[:-1], fd, rtol=1e-5, atol=1e-5 * np.abs(fd).max())


@pytest.mark.parametrize("model_name", ["MultiTaskGP", "CoregGP"])
@pytest.mark.parametrize("acq_name", ["EI", "UCB"])
def test_optimize_acq_end_to_end(ctx, model_name, acq_name, monkeypatch):
    run_and_check(ctx, lcm_models(ctx)[model_name], acq_name, monkeypatch)


def test_posterior_grad_of_the_model_matches_the_oracle(ctx):
    """_LCMModel._posterior_grad: the library's rows for every draw, the task column's entries 0"""
    model = lcm_models(ctx)["MultiTaskGP"]
    samples = model.get_samples()
    Xn = np.c_[np.random.default_rng(3).uniform(-2, 2, (4, 2)), [0, 1, 1, 0]]
    mean, var, dmean, dvar = model._posterior_grad(Xn, samples, True, False)
    assert dmean.shape == dvar.shape == (3, 4, 3) and np.all(dmean[..., -1] == 0) and np.all(dvar[..., -1] == 0)
    for s in range(3):
        ps = {k: np.asarray(v)[s] for k, v in samples.items()}
        ps["k_scale"] = np.asarray(ps["k_scale"])
        ps["period"] = None
        ref = oracle_grad(model.X_train, model.y_train, Xn, ps, "RBF", False, 2)
        for got, r in zip((mean[s], var[s], dmean[s], dvar[s]), ref):
            assert_close(got, r, 1e-7, f"draw {s}")


def test_optimize_acq_after_a_short_nuts_fit(ctx, monkeypatch):
    from gpax_b200 import MultiTaskGP
    X, y = bo_data()
    model = MultiTaskGP(2, "RBF", num_latents=2, num_tasks=2, ctx=ctx)
    model.fit(0, X, y, num_warmup=50, num_samples=50, progress_bar=False, print_summary=False)
    run_and_check(ctx, model, "EI", monkeypatch, task=0.0)
