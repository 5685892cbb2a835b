"""GPU: the launch count a call reports (b2gp_timing::launches, `last_timing()["launches"]`, bench.py's gpu_launches) is
the number of kernels the CUDA profiler sees that call run.

torch.profiler with CUDA activities records every kernel of the process, those queued by libb200gp.so through ctypes
included, so it is an independent count.  Each test runs on a context of its own; the rowdot cases also check the count
that follows from the entry point's code (one reduction, plus one accumulation per requested output)."""
import collections

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def profiled_kernels(fn):
    """names of the kernels the CUDA profiler recorded while fn() ran"""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]


def assert_launches_match_profiler(ctx, fn):
    names = profiled_kernels(fn)
    launches = ctx.last_timing()["launches"]
    assert names, "torch.profiler recorded no kernel of the call: it does not see libb200gp.so's launches"
    assert launches == len(names), f"reported {launches} launches, the profiler saw {len(names)}: {collections.Counter(names)}"
    return launches


def gp_data(rng, N, P, d=2):
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(4 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    return X, y, rng.uniform(0, 1, (P, d))


THETA = np.array([0.3, 0.4, 1.0, 0.05, 1.0])   # lengthscale[2], k_scale, noise, period


@pytest.mark.parametrize("ozaki", [0, 7])
def test_posterior_all_outputs(ctx, ozaki):
    # N >= tall_min: under ozaki 7 the factorisation takes the tall-panel int8 route; S > streams queues the draws from
    # one host thread per slot
    rng = np.random.default_rng(1)
    X, y, Xn = gp_data(rng, 2100, 96)
    S, n = 3, 2
    theta = np.tile(THETA, (S, 1))
    eps = rng.standard_normal((S, n, 96))
    ctx.set_option("ozaki", ozaki)
    out = {}
    assert_launches_match_profiler(ctx, lambda: out.update(ctx.posterior("RBF", X, y, Xn, theta, want=("mean", "var", "cov"), eps=eps)))
    assert (out["info"] == 0).all()


def test_sparse_posterior(ctx):
    rng = np.random.default_rng(2)
    X, y, Xn = gp_data(rng, 900, 70)
    Xu = X[:64]
    out = {}
    assert_launches_match_profiler(ctx, lambda: out.update(ctx.sparse_posterior("Matern", Xu, X, y, Xn, THETA, want=("mean", "var", "cov"))))
    assert out["info"] == 0


def test_sparse_elbo(ctx):
    rng = np.random.default_rng(3)
    X, y, _ = gp_data(rng, 600, 1)
    out = []
    assert_launches_match_profiler(ctx, lambda: out.extend(ctx.sparse_elbo("RBF", X[:48], X, y, THETA)))
    assert out[3] == 0 and np.isfinite(out[0])


def test_mll_with_gradient(ctx):
    rng = np.random.default_rng(4)
    X, y, _ = gp_data(rng, 500, 1)
    out = []
    assert_launches_match_profiler(ctx, lambda: out.extend(ctx.mll("Matern", X, y, THETA, want_grad=True)))
    assert out[3] == 0 and np.isfinite(out[1]).all()


def test_mvn_sample(ctx):
    rng = np.random.default_rng(5)
    S, P, n = 2, 80, 3
    B = rng.standard_normal((S, P, P))
    cov = B @ B.transpose(0, 2, 1) / P + np.eye(P)
    mean = rng.standard_normal((S, P))
    assert_launches_match_profiler(ctx, lambda: ctx.mvn_sample(mean, cov, rng.standard_normal((S, n, P))))


def test_acq_moments(ctx):
    rng = np.random.default_rng(6)
    mean, var = rng.standard_normal((4, 200)), rng.uniform(0.1, 1.0, (4, 200))
    assert assert_launches_match_profiler(ctx, lambda: ctx.acq_moments("EI", mean, var)) == 2   # best value, then EI


def test_gemm_nt(ctx):
    rng = np.random.default_rng(7)
    A, B = rng.standard_normal((300, 200)), rng.standard_normal((250, 200))
    assert_launches_match_profiler(ctx, lambda: ctx.gemm_nt(A, B))


def test_potrf(ctx):
    rng = np.random.default_rng(8)
    B = rng.standard_normal((700, 700))
    out = []
    assert_launches_match_profiler(ctx, lambda: out.extend(ctx.potrf(B @ B.T / 700 + np.eye(700))))
    assert out[1] == 0


@pytest.mark.parametrize("dot,nrm", [(True, True), (True, False), (False, True)])
def test_rowdot(ctx, dot, nrm):
    rng = np.random.default_rng(9)
    R, w = rng.standard_normal((120, 75)), rng.standard_normal(75)
    dR, dw, ddot, dnrm = ctx.to_device(R), ctx.to_device(w), ctx.alloc(120), ctx.alloc(120)

    def call():
        ctx._check(ctx.lib.b2gp_rowdot(ctx.h, 120, 75, dR.ptr, 75, dw.ptr, 1.0, ddot.ptr if dot else None, dnrm.ptr if nrm else None, 0))

    assert assert_launches_match_profiler(ctx, call) == 1 + dot + nrm
    if dot:
        np.testing.assert_allclose(ddot.download(), R @ w, rtol=1e-12)
    if nrm:
        np.testing.assert_allclose(dnrm.download(), (R * R).sum(1), rtol=1e-12)
