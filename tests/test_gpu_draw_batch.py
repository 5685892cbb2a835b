"""GPU: multi-draw posteriors factored in lock-step groups on the fp64 tall-panel route (draw_batch, DESIGN.md 4.2).

Within a draw the batched kernels issue the same DMMA instructions in the same k order as the per-draw route, so every
output must be bit-identical to draw_batch = 1."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_TALL = 8192


@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    c.set_option("streams", 8)
    yield c
    c.close()


def counted(ctx, fn):
    before = ctx.path_counts()
    out = fn()
    after = ctx.path_counts()
    return out, {k: after[k] - before[k] for k in after}


def inputs(N, P, S, d=2, seed=0):
    rng = np.random.default_rng(seed + N + P + S)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    theta = np.column_stack([rng.uniform(0.2, 0.4, (S, d)), rng.uniform(0.8, 1.2, S), rng.uniform(0.03, 0.08, S),
                             rng.uniform(0.7, 1.1, S)])
    return X, y, Xn, theta


def both(ctx, fn, **opts):
    """fn() under draw_batch = 1 and under `opts` (default: the route's own group size), with the counter deltas"""
    with ctx.options(draw_batch=1):
        ref, c1 = counted(ctx, fn)
    with ctx.options(**opts):
        got, c = counted(ctx, fn)
    return ref, got, c1, c


def group_size(S, streams, draw_batch=0):
    """the library's rule (posterior_impl): two groups of up to 4 in flight, else one draw per group"""
    n = min(S, streams)
    if draw_batch:
        return min(draw_batch, n)
    B = min(4, n // 2)
    return B if B >= 2 else 1


def batched_groups(S, B):
    return 0 if B == 1 else S // B + (S % B > 1)


def assert_same(ref, got, names):
    for k in names:
        assert ref[k] is not None and np.array_equal(ref[k], got[k], equal_nan=True), k
    assert np.array_equal(ref["info"], got["info"])


@pytest.mark.parametrize("S,streams,draw_batch", [(2, 8, 2), (3, 8, 3), (8, 8, 0), (11, 4, 0), (6, 8, 0), (7, 8, 0), (5, 8, 4),
                                                 (8, 2, 0), (3, 8, 0)])
def test_bit_identical_draw_counts(ctx, S, streams, draw_batch):
    """explicit group sizes and the route's own choice (two groups in flight, or the per-draw route on 2 streams)"""
    X, y, Xn, theta = inputs(N_TALL, 300, S)
    ctx.set_option("streams", streams)
    fn = lambda: ctx.posterior("RBF", X, y, Xn, theta, want=("mean", "var"))
    ref, got, c1, c = both(ctx, fn, draw_batch=draw_batch)
    assert_same(ref, got, ("mean", "var"))
    assert (got["info"] == 0).all()
    B = group_size(S, streams, draw_batch)
    assert c["potrf_tall_batch"] == batched_groups(S, B) and c1["potrf_tall_batch"] == 0, (B, c)
    assert c["potrf_tall_fp64"] == c1["potrf_tall_fp64"] == S
    assert c["panel_solve"] == c1["panel_solve"] == S * (N_TALL // 1024)
    if B > 1:
        assert c["potrf_diag"] < c1["potrf_diag"] and c["gemm_tma"] + c["gemm_nt"] < c1["gemm_tma"] + c1["gemm_nt"], (c, c1)
    else:
        assert c == c1


@pytest.mark.parametrize("B", [2, 4, 8])
@pytest.mark.parametrize("kname", ["RBF", "Matern", "Periodic"])
def test_bit_identical_kernels_and_group_sizes(ctx, kname, B):
    X, y, Xn, theta = inputs(N_TALL, 1025, 8)
    eps = np.random.default_rng(1).standard_normal((8, 2, 1025))
    ref, got, _, c = both(ctx, lambda: ctx.posterior(kname, X, y, Xn, theta, want=("mean", "var", "cov"), eps=eps), draw_batch=B)
    assert_same(ref, got, ("mean", "var", "cov", "y_sampled"))
    assert c["potrf_tall_batch"] == 8 // B


@pytest.mark.parametrize("P", [1, 300, 1025])
def test_bit_identical_ragged_N(ctx, P):
    """N = 3000 with tall_min_fp64 lowered: a ragged last panel and leaf, P + 1 rows not a multiple of 128"""
    X, y, Xn, theta = inputs(3000, P, 5)
    with ctx.options(tall_min_fp64=2048):
        ref, got, _, c = both(ctx, lambda: ctx.posterior("Matern", X, y, Xn, theta, want=("mean", "var", "cov")))
    assert_same(ref, got, ("mean", "var", "cov"))
    assert c["potrf_tall_batch"] == 2


def test_bit_identical_grad(ctx):
    X, y, Xn, theta = inputs(N_TALL, 64, 6)
    ref, got, _, c = both(ctx, lambda: ctx.posterior_grad("RBF", X, y, Xn, theta))
    assert_same(ref, got, ("mean", "var", "dmean", "dvar"))
    assert c["potrf_tall_batch"] == 2


def test_bit_identical_nngp(ctx):
    X, y, Xn, _ = inputs(N_TALL, 200, 4)
    theta = np.column_stack([np.full((4, 2), 2.0), np.linspace(1.0, 1.5, 4), np.full(4, 0.05), np.full(4, 0.1)])
    ref, got, _, c = both(ctx, lambda: ctx.posterior("NNGP_relu", X, y, Xn, theta, want=("mean", "var")))
    assert_same(ref, got, ("mean", "var"))
    assert c["potrf_tall_batch"] == 2


def test_failed_draw_is_isolated(ctx):
    """a draw with a negative noise (K not positive definite) inside a group: its info is set and its outputs are NaN,
    the other draws are bit-identical to the same call without it"""
    X, y, Xn, theta = inputs(N_TALL, 100, 4)
    bad = theta.copy()
    bad[1, 2 + 1] = -50.0
    ok = ctx.posterior("RBF", X, y, Xn, theta, want=("mean", "var"))
    got, c = counted(ctx, lambda: ctx.posterior("RBF", X, y, Xn, bad, want=("mean", "var")))
    assert c["potrf_tall_batch"] == 2
    assert got["info"][1] != 0 and np.isnan(got["mean"][1]).all() and np.isnan(got["var"][1]).all()
    for s in (0, 2, 3):
        assert got["info"][s] == 0
        assert np.array_equal(got["mean"][s], ok["mean"][s]) and np.array_equal(got["var"][s], ok["var"][s])


def test_single_draw_never_batched(ctx):
    X, y, Xn, theta = inputs(N_TALL, 100, 1)
    _, c = counted(ctx, lambda: ctx.posterior("RBF", X, y, Xn, theta, want=("mean", "var")))
    assert c["potrf_tall_batch"] == 0 and c["potrf_tall_fp64"] == 1


def test_fewer_launches(ctx):
    X, y, Xn, theta = inputs(N_TALL, 1000, 8)
    fn = lambda: ctx.posterior("RBF", X, y, Xn, theta, want=("mean", "var"), timing=True)
    with ctx.options(draw_batch=1):
        l1 = fn()["timing"]["launches"]
    lb = fn()["timing"]["launches"]
    assert lb < l1 / 2, (lb, l1)


def test_fit_then_predict_device_memory():
    """a likelihood evaluation and then an 8-draw posterior on one context hold no more device memory than the posterior
    alone plus the likelihood's own N x N scratch (K^{-1} and dK products, slot 0's Vt and cov), and the posterior at most
    the per-draw buffers of 8 slots: slot 0's factor matrix of the likelihood is the front of the posterior's draw regions"""
    import torch
    from gpax_b200 import _ffi
    N, P, S = N_TALL, 1000, 8
    X, y, Xn, theta = inputs(N, P, S)
    torch.cuda.mem_get_info(0)

    def used(run):
        free0 = torch.cuda.mem_get_info(0)[0]
        c = _ffi.Context(0)
        c.set_option("streams", 8)
        try:
            run(c)
            return free0 - torch.cuda.mem_get_info(0)[0]
        finally:
            c.close()

    post = lambda c: c.posterior("RBF", X, y, Xn, theta, want=("mean", "var"))
    u_post = used(post)
    u_both = used(lambda c: (c.mll("RBF", X, y, theta[0]), post(c)))
    slack = 64 << 20   # staging, small scratch, allocation rounding
    ld = -(-N // 8) * 8
    assert u_both <= u_post + 2 * N * ld * 8 + slack, (u_both, u_post)
    per_draw = (N + P + 1) * ld * 8 + -(-N // 128) * 128 * 128 * 8 + 2 * 1024 * 1024 * 8   # A | Linv | panel scratch
    assert u_post <= S * per_draw + slack, (u_post, S * per_draw)
