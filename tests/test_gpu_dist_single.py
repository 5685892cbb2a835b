"""GPU, one device: the multi-GPU entry points and their building blocks against the oracle.

  1. b2gp_dist_sparse_posterior on one rank: bit-identical to b2gp_sparse_posterior (the same device functions on the same
     stream, no all-reduce), at the bench's c5 shape too; against the oracle; failure signs of info; refusals.
  2. the sharded statistics (b2gp_sparse_partial per shard, summed here, b2gp_sparse_finish) against the oracle on the
     full training set -- the algebra the in-library all-reduce relies on.
  3. b2gp_dist_posterior on a 1 x 1 grid against the oracle at the shapes where the block-cyclic bookkeeping changes:
     one or two tile rows, P = 1, nb - 1, nb, nb + 1 and P > N, noiseless, mean only, every plane count, both list widths.
  4. b2gp_potrf_inv, b2gp_trsm_inv, b2gp_rowdot, b2gp_copy2d directly, and GpuOps against the NumPy stand-in
     (tests/dist_helpers.py) that the CPU gloo tests run in their place.
Everything that calls b2gp_dist_init runs in ONE worker process (tests/dist_single_worker.py), reaped here."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import scipy.linalg as sla

import oracle
from conftest import ROOT, assert_close
from dist_single_worker import SENTINEL, c5_problem, dense_problem, sparse_problem

pytestmark = pytest.mark.gpu

RTOL = 1e-9          # the parity bar at cond <= 1e5, scaled by cond / 1e5 beyond (test_gpu_paths.py)
ERR_ARG = -1


def params_of(theta, d):
    return {"k_length": theta[:d], "k_scale": theta[d], "noise": theta[d + 1], "period": theta[d + 2]}


def run_worker(cases, timeout=900):
    """all cases in one worker process; the process is killed and reaped whatever happens"""
    with tempfile.TemporaryDirectory() as td:
        with open(os.path.join(td, "cases.json"), "w") as f:
            json.dump(cases, f)
        env = dict(os.environ, RANK="0", WORLD_SIZE="1", LOCAL_RANK="0")
        p = subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "dist_single_worker.py"), os.path.join(td, "cases.json"), td],
                             env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        try:
            log = p.communicate(timeout=timeout)[0]
        finally:
            if p.poll() is None:
                p.kill()
            p.communicate()
        assert p.returncode == 0, log[-4000:]
        return {c["id"]: dict(np.load(os.path.join(td, c["id"] + ".npz"))) for c in cases}


# ------------------------------------------------------------------ cases of the worker
# dense: (N, P, nb, kernel, ozaki, oz_cluster, extra).  The largest first: every later case reuses its buffers.
# ozaki None: the option is not touched (library default 0, which means "planes from the conditioning" on this path).
DENSE = {
    "T3_nb1024_P_nb+1": (3072, 1025, 1024, "RBF", -1, 2, {}),
    "T2_nb1024_P_nb": (2048, 1024, 1024, "Matern", 0, 1, {}),
    "T1_nb1024_P1": (1024, 1, 1024, "Periodic", 7, 1, {}),
    "T4_nb256_P_gt_N": (1024, 1500, 256, "Matern", 6, 2, {}),
    "T3_nb256_P_nb+1_noiseless": (768, 257, 256, "RBF", 7, 1, {"noiseless": True}),
    "T2_nb256_P_nb": (512, 256, 256, "Periodic", None, None, {}),
    "T1_nb256_P_nb-1_mean_only": (256, 255, 256, "Matern", -1, 1, {"want_var": False}),
    "T5_nb128_P_nb+1_noiseless": (640, 129, 128, "Matern", 7, 2, {"noiseless": True}),
    "T3_nb128_P_nb": (384, 128, 128, "RBF", 6, 1, {}),
    "T2_nb128_P_nb-1": (256, 127, 128, "Periodic", 7, 2, {}),
    "T2_nb128_P_gt_N_noiseless": (256, 700, 128, "RBF", -1, 1, {"noiseless": True}),
    "T1_nb128_P1": (128, 1, 128, "Matern", 7, 1, {}),
    "not_pd": (1024, 300, 256, "Matern", 7, 2, {"noise": -0.05}),
    "after_not_pd": (1024, 300, 256, "Matern", 7, 2, {}),
}
# sparse: (N, M, P, kernel, ozaki, extra); "bits": also the single-GPU entry point on the same context
SPARSE = {}
for _k in ("RBF", "Matern", "Periodic"):
    for _oz in (0, 7):
        SPARSE[f"small_{_k}_oz{_oz}"] = (1500, 96, 70, _k, _oz, {"bits": True})
        SPARSE[f"medium_{_k}_oz{_oz}"] = (5000, 300, 300, _k, _oz, {"bits": True})
SPARSE.update({
    "small_noiseless": (1500, 96, 70, "Matern", 0, {"noiseless": True}),
    "medium_noiseless": (5000, 300, 300, "RBF", 7, {"noiseless": True}),
    "small_mean_only": (1500, 96, 70, "RBF", 0, {"want_var": False}),
    "Kuu_not_pd": (1500, 96, 70, "RBF", 0, {"k_scale": -1.0}),
    "negative_noise": (1500, 96, 70, "Matern", 0, {"noise": -0.05}),
    "after_failures": (1500, 96, 70, "Periodic", 0, {}),
})
_OUT_MEAN, _OUT_VAR, _OUT_COV, _OUT_SAMPLE, _DEV = 1 << 4, 1 << 5, 1 << 6, 1 << 7, 1 << 0
REFUSE = {
    "dense_N_not_multiple_of_nb": {"entry": "dense", "N": 300, "nb": 128},
    "dense_nb64": {"entry": "dense", "N": 256, "nb": 64},
    "dense_nb192": {"entry": "dense", "N": 384, "nb": 192},
    "dense_nb2048": {"entry": "dense", "N": 2048, "nb": 2048},
    "dense_kind3": {"entry": "dense", "kind": 3},
    "dense_kind4": {"entry": "dense", "kind": 4},
    "dense_out_cov": {"entry": "dense", "flags": _OUT_MEAN | _OUT_COV},
    "dense_out_sample": {"entry": "dense", "flags": _OUT_MEAN | _OUT_SAMPLE},
    "dense_device_ptrs": {"entry": "dense", "flags": _OUT_MEAN | _DEV},
    "sparse_out_cov": {"entry": "sparse", "flags": _OUT_MEAN | _OUT_COV},
    "sparse_device_ptrs": {"entry": "sparse", "flags": _OUT_MEAN | _DEV},
    "sparse_kind3": {"entry": "sparse", "kind": 3},
    "sparse_kind4": {"entry": "sparse", "kind": 4},
    "sparse_d65": {"entry": "sparse", "d": 65},
}


def _cases():
    cases = []
    for cid, (N, P, nb, kernel, oz, cl, extra) in DENSE.items():
        cases.append(dict(id="dense_" + cid, op="dense", N=N, P=P, nb=nb, kernel=kernel, ozaki=oz, oz_cluster=cl, **extra))
    cases.append(dict(id="sparse_c5", op="sparse", c5=True, kernel="Matern", bits=True))
    for cid, (N, M, P, kernel, oz, extra) in SPARSE.items():
        cases.append(dict(id="sparse_" + cid, op="sparse", N=N, M=M, P=P, kernel=kernel, ozaki=oz, **extra))
    for cid, kw in REFUSE.items():
        cases.append(dict(id="refuse_" + cid, op="refuse", **kw))
    # the same context still works after the refusals
    cases.append(dict(id="dense_after_refusals", op="dense", N=512, P=200, nb=128, kernel="RBF", ozaki=7, oz_cluster=2))
    cases.append(dict(id="sparse_after_refusals", op="sparse", N=1500, M=96, P=70, kernel="RBF", ozaki=0))
    return cases


@pytest.fixture(scope="module")
def results():
    return run_worker(_cases())


# ------------------------------------------------------------------ 1. b2gp_dist_sparse_posterior on one rank
def sparse_oracle(case):
    N, M, P, kernel, oz, extra = case
    X, y, Xu, Xn, theta = sparse_problem(N, M, P, 2, kernel, extra.get("k_scale", 1.0), extra.get("noise", 0.05))
    p = params_of(theta, 2)
    rmean, rcov = oracle.sparse_posterior(X, y, Xu, Xn, p, kernel, noiseless=extra.get("noiseless", False), jitter=1e-5)
    k = oracle.get_kernel(kernel)
    Kuu = k(Xu, Xu, p, jitter=1e-5)
    W = sla.solve_triangular(np.linalg.cholesky(Kuu), k(Xu, X, p, jitter=0.0), lower=True)
    ev_u, ev_k = np.linalg.eigvalsh(Kuu), np.linalg.eigvalsh(W @ W.T / p["noise"] + np.eye(M))
    cond = max(ev_u[-1] / ev_u[0], ev_k[-1] / ev_k[0])
    return rmean, np.diag(rcov), RTOL * max(1.0, cond / 1e5), cond


@pytest.mark.parametrize("cid", [c for c in SPARSE if "bits" in SPARSE[c][5]] + ["c5"])
def test_dist_sparse_one_rank_is_bit_identical_to_single_gpu(results, cid):
    r = results["sparse_" + cid]
    assert r["info"] == 0 and r["one_info"] == 0
    assert np.array_equal(r["mean"], r["one_mean"]), f"{cid}: mean differs from b2gp_sparse_posterior"
    assert np.array_equal(r["var"], r["one_var"]), f"{cid}: var differs from b2gp_sparse_posterior"
    if cid == "c5":
        X, y, Xu, Xn, theta = c5_problem()
        assert r["mean"].shape == (Xn.shape[0],) and np.isfinite(r["mean"]).all() and (r["var"] > 0).all()


@pytest.mark.parametrize("cid", [c for c in SPARSE if SPARSE[c][5].get("bits") or not set(SPARSE[c][5]) & {"k_scale", "noise"}])
def test_dist_sparse_one_rank_vs_oracle(results, cid):
    r = results["sparse_" + cid]
    rmean, rvar, tol, cond = sparse_oracle(SPARSE[cid])
    what = f"{cid}: cond <= {cond:.1e}"
    assert r["info"] == 0, what
    assert_close(r["mean"], rmean, tol, "mean " + what)
    if SPARSE[cid][5].get("want_var", True):
        assert_close(r["var"], rvar, tol, "var " + what)
    else:
        assert (r["var"] == SENTINEL).all(), "a mean-only call wrote var"


def test_dist_sparse_one_rank_failures(results):
    r = results["sparse_Kuu_not_pd"]            # chol(Kuu + jitter I) fails: info > 0
    assert r["info"] > 0 and np.isnan(r["mean"]).all() and np.isnan(r["var"]).all()
    r = results["sparse_negative_noise"]        # chol(W W^T / noise + I) fails: info < 0
    assert r["info"] < 0 and np.isnan(r["mean"]).all() and np.isnan(r["var"]).all()
    for cid in ("after_failures",):
        r = results["sparse_" + cid]
        rmean, rvar, tol, cond = sparse_oracle(SPARSE[cid])
        assert r["info"] == 0
        assert_close(r["mean"], rmean, tol, "mean after failures")
        assert_close(r["var"], rvar, tol, "var after failures")


# ------------------------------------------------------------------ 3. b2gp_dist_posterior on a 1 x 1 grid
def dense_oracle(N, P, kernel, noise, noiseless):
    X, y, Xn, theta = dense_problem(N, P, kernel, noise)
    p = params_of(theta, 2)
    rmean, rvar = oracle.exact_posterior_chol(X, y, Xn, p, kernel, noiseless=noiseless, diag_only=True, jitter=1e-6)
    cond = (N * p["k_scale"] + p["noise"] + 1e-6) / (p["noise"] + 1e-6)      # Gershgorin: every entry of k <= k_scale
    return rmean, rvar, RTOL * max(1.0, cond / 1e5)


@pytest.mark.parametrize("cid", [c for c in DENSE if c != "not_pd"])
def test_dist_posterior_one_rank_vs_oracle(results, cid):
    N, P, nb, kernel, oz, cl, extra = DENSE[cid]
    r = results["dense_" + cid]
    rmean, rvar, tol = dense_oracle(N, P, kernel, extra.get("noise", 0.05), extra.get("noiseless", False))
    what = f"{cid} (N={N} P={P} nb={nb} {kernel} ozaki={oz} oz_cluster={cl})"
    assert r["info"] == 0, what
    assert_close(r["mean"], rmean, tol, "mean " + what)
    if extra.get("want_var", True):
        assert_close(r["var"], rvar, tol, "var " + what)
    else:
        assert (r["var"] == SENTINEL).all(), "a mean-only call wrote var"


def test_dist_posterior_not_positive_definite_then_recovers(results):
    r = results["dense_not_pd"]
    assert r["info"] > 0 and np.isnan(r["mean"]).all() and np.isnan(r["var"]).all()
    r = results["dense_after_not_pd"]
    rmean, rvar, tol = dense_oracle(1024, 300, "Matern", 0.05, False)
    assert r["info"] == 0
    assert_close(r["mean"], rmean, tol, "mean after a failed call")
    assert_close(r["var"], rvar, tol, "var after a failed call")


@pytest.mark.parametrize("cid", list(REFUSE))
def test_dist_entry_points_refuse_bad_arguments(results, cid):
    r = results["refuse_" + cid]
    assert r["rc"] == ERR_ARG and str(r["msg"]), cid
    assert (r["mean"] == SENTINEL).all() and (r["var"] == SENTINEL).all() and r["info"] == 7, f"{cid}: refused call wrote output"


def test_context_works_after_refusals(results):
    r = results["dense_after_refusals"]
    rmean, rvar, tol = dense_oracle(512, 200, "RBF", 0.05, False)
    assert r["info"] == 0
    assert_close(r["mean"], rmean, tol, "dense mean after refusals")
    assert_close(r["var"], rvar, tol, "dense var after refusals")
    r = results["sparse_after_refusals"]
    rmean, rvar, tol, _ = sparse_oracle((1500, 96, 70, "RBF", 0, {}))
    assert r["info"] == 0
    assert_close(r["mean"], rmean, tol, "sparse mean after refusals")


def test_dist_entry_points_refuse_a_context_without_dist_init():
    from gpax_b200 import _ffi
    ctx = _ffi.Context(0)
    try:
        X, y, Xn, theta = dense_problem(256, 10, "RBF")
        mean, var, info = np.full(10, SENTINEL), np.full(10, SENTINEL), C.c_int(7)
        rc = ctx.lib.b2gp_dist_posterior(ctx.h, 0, _ffi._ptr(X), 256, _ffi._ptr(y), _ffi._ptr(Xn), 10, 2, _ffi._ptr(theta), 0, 1e-6, 128,
                                         _OUT_MEAN | _OUT_VAR, _ffi._ptr(mean), _ffi._ptr(var), C.byref(info), None)
        assert rc == ERR_ARG and b"b2gp_dist_init" in ctx.lib.b2gp_last_error(ctx.h)
        rc = ctx.lib.b2gp_dist_sparse_posterior(ctx.h, 0, _ffi._ptr(X[:32]), 32, _ffi._ptr(X), 256, _ffi._ptr(y), _ffi._ptr(Xn), 10, 2,
                                                _ffi._ptr(theta), 0, 1e-5, _OUT_MEAN | _OUT_VAR, _ffi._ptr(mean), _ffi._ptr(var),
                                                C.byref(info), None)
        assert rc == ERR_ARG and b"b2gp_dist_init" in ctx.lib.b2gp_last_error(ctx.h)
        assert (mean == SENTINEL).all() and (var == SENTINEL).all() and info.value == 7
    finally:
        ctx.close()


# ------------------------------------------------------------------ 2. the sharded statistics, summed here
@pytest.fixture
def ctx():
    from gpax_b200 import _ffi
    c = _ffi.Context(0)
    yield c
    c.close()


def sharded_posterior(ctx, kernel, Xu, X, y, Xn, theta, bounds, noiseless=False, ldk=None, want_cov=True):
    """b2gp_sparse_partial per shard [lo, hi), Kpart / cpart summed on the host, b2gp_sparse_finish (device arrays)"""
    from gpax_b200 import _ffi
    M, d = Xu.shape
    P = Xn.shape[0]
    ldk = ldk or M
    th = np.ascontiguousarray(theta, dtype=np.float64)
    dXu, dXn = ctx.to_device(Xu), ctx.to_device(Xn)
    Kp, cp = ctx.alloc((M, ldk)), ctx.alloc(M)
    Ksum, csum, infos = np.zeros((M, ldk)), np.zeros(M), []
    for lo, hi in bounds:
        dX, dy = ctx.to_device(X[lo:hi]), ctx.to_device(y[lo:hi])
        info = C.c_int(7)
        ctx._check(ctx.lib.b2gp_sparse_partial(ctx.h, _ffi.KIND[kernel], dXu.ptr, M, dX.ptr, hi - lo, dy.ptr, d, _ffi._ptr(th), 1e-5,
                                               Kp.ptr, ldk, cp.ptr, C.byref(info)))
        infos.append(info.value)
        Ksum += np.tril(Kp.download())       # the lower triangle is the statistic (b200gp.h); the library reads only it
        csum += cp.download()
    dK, dc = ctx.to_device(Ksum), ctx.to_device(csum)
    dmean, dvar, dcov = ctx.alloc(P), ctx.alloc(P), ctx.alloc((P, P))
    info = C.c_int(7)
    flags = _OUT_MEAN | _OUT_VAR | (_OUT_COV if want_cov else 0)
    ctx._check(ctx.lib.b2gp_sparse_finish(ctx.h, _ffi.KIND[kernel], dXu.ptr, M, dK.ptr, ldk, dc.ptr, dXn.ptr, P, d, _ffi._ptr(th),
                                          int(noiseless), 1e-5, flags, dmean.ptr, dvar.ptr, dcov.ptr if want_cov else None,
                                          C.byref(info)))
    return {"mean": dmean.download(), "var": dvar.download(), "cov": dcov.download() if want_cov else None,
            "partial_info": infos, "info": info.value, "Ksum": Ksum, "csum": csum}


SHARDS = {
    "equal": lambda N, M: [(i * N // 4, (i + 1) * N // 4) for i in range(4)],
    "unequal": lambda N, M: [(0, 1), (1, 700), (700, 701), (701, N)],             # with two 1-point shards
    "smaller_than_M": lambda N, M: [(lo, min(N, lo + M // 2)) for lo in range(0, N, M // 2)],
    "one_shard_ldk_gt_M": lambda N, M: [(0, N)],
}


@pytest.mark.parametrize("shards", list(SHARDS))
@pytest.mark.parametrize("noiseless", [False, True])
def test_sharded_statistics_sum_to_the_full_set_posterior(ctx, shards, noiseless):
    N, M, P, kernel = 1500, 96, 70, "Matern"
    X, y, Xu, Xn, theta = sparse_problem(N, M, P, 2, kernel)
    bounds = SHARDS[shards](N, M)
    assert bounds[0][0] == 0 and bounds[-1][1] == N and all(a[1] == b[0] for a, b in zip(bounds, bounds[1:]))
    ldk = M + 13 if shards == "one_shard_ldk_gt_M" else None
    out = sharded_posterior(ctx, kernel, Xu, X, y, Xn, theta, bounds, noiseless, ldk)
    rmean, _, tol, cond = sparse_oracle((N, M, P, kernel, 0, {"noiseless": noiseless}))
    _, rcov = oracle.sparse_posterior(X, y, Xu, Xn, params_of(theta, 2), kernel, noiseless=noiseless, jitter=1e-5)
    what = f"{len(bounds)} shards ({shards}), noiseless={noiseless}, cond <= {cond:.1e}"
    assert out["partial_info"] == [0] * len(bounds) and out["info"] == 0, what
    assert_close(out["mean"], rmean, tol, "mean " + what)
    assert_close(out["var"], np.diag(rcov), tol, "var " + what)
    assert_close(out["cov"], rcov, tol, "cov " + what)
    # the unsharded entry point: the same posterior, summed in another order
    one = ctx.sparse_posterior(kernel, Xu, X, y, Xn, theta, noiseless=noiseless, jitter=1e-5, want=("mean", "var", "cov"))
    assert_close(out["mean"], one["mean"], tol, "mean vs b2gp_sparse_posterior " + what)
    assert_close(out["cov"], one["cov"], tol, "cov vs b2gp_sparse_posterior " + what)


def test_sharded_statistics_failure_signs(ctx):
    N, M, P = 1500, 96, 70
    bounds = [(0, 600), (600, N)]
    X, y, Xu, Xn, theta = sparse_problem(N, M, P, 2, "RBF", k_scale=-1.0)       # chol(Kuu + jitter I) fails
    out = sharded_posterior(ctx, "RBF", Xu, X, y, Xn, theta, bounds)
    assert all(i > 0 for i in out["partial_info"]) and out["info"] > 0
    assert np.isnan(out["mean"]).all() and np.isnan(out["var"]).all() and np.isnan(out["cov"]).all()
    X, y, Xu, Xn, theta = sparse_problem(N, M, P, 2, "RBF", noise=-0.05)        # chol(sum W W^T / noise + I) fails
    out = sharded_posterior(ctx, "RBF", Xu, X, y, Xn, theta, bounds)
    assert out["partial_info"] == [0, 0] and out["info"] < 0
    assert np.isnan(out["mean"]).all() and np.isnan(out["var"]).all() and np.isnan(out["cov"]).all()


# ------------------------------------------------------------------ 4. building blocks
def spd(rng, n, cond=1e3):
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q * np.geomspace(1.0, cond, n)) @ Q.T
    return (A + A.T) / 2


def potrf_inv(ctx, A, lda):
    """b2gp_potrf_inv on A stored with leading dimension lda and two extra rows; returns (stored matrix, Linv blocks, info)"""
    n = A.shape[0]
    store = np.full((n + 2, lda), 777.0)
    store[:n, :n] = A
    dA, dL = ctx.to_device(store), ctx.alloc((-(-n // 128), 128, 128))
    info = C.c_int(-7)
    ctx._check(ctx.lib.b2gp_potrf_inv(ctx.h, n, dA.ptr, lda, dL.ptr, C.byref(info)))
    return dA.download(), dL.download(), info.value


@pytest.mark.parametrize("n", [1, 127, 128, 129, 300, 640])
def test_potrf_inv_factor_and_exported_block_inverses(ctx, n):
    rng = np.random.default_rng(n)
    A = spd(rng, n)
    lda = n + 3
    got, blocks, info = potrf_inv(ctx, A, lda)
    assert info == 0
    L = sla.cholesky(A, lower=True)
    assert_close(np.tril(got[:n, :n]), L, 1e-12, f"L, n={n}")
    assert (got[:n, n:] == 777.0).all() and (got[n:] == 777.0).all(), "wrote outside the n x n matrix"
    # potrf_diag_kernel writes inv(L_bb) of each 128-wide diagonal block row-major with leading dimension 128, lower
    # triangular (zero above the diagonal); a ragged last block is valid in its leading (n mod 128) square only
    for b in range(blocks.shape[0]):
        lo, hi = 128 * b, min(n, 128 * (b + 1))
        w = hi - lo
        ref = sla.solve_triangular(L[lo:hi, lo:hi], np.eye(w), lower=True)
        assert_close(blocks[b, :w, :w], ref, 1e-11, f"inv(L_bb), block {b}, n={n}")
        assert not np.triu(blocks[b, :w, :w], 1).any(), "upper triangle of an exported inverse"


@pytest.mark.parametrize("n,j", [(1, 0), (129, 0), (300, 200), (640, 129), (640, 639)])
def test_potrf_inv_reports_the_first_bad_pivot(ctx, n, j):
    A = spd(np.random.default_rng(n + j), n)
    L = np.linalg.cholesky(A)
    A[j, j] -= L[j, j] ** 2 + 1.0          # pivot j becomes sqrt(-1); the pivots before it are untouched
    assert sla.lapack.dpotrf(A, lower=1)[1] == j + 1
    _, _, info = potrf_inv(ctx, A, n + 8)
    assert info == j + 1


@pytest.mark.parametrize("ozaki", [0, 7])
@pytest.mark.parametrize("n", [128, 300, 640])
@pytest.mark.parametrize("nrhs", [0, 1, 1100])
def test_trsm_inv_solves_with_the_exported_inverses(ctx, n, nrhs, ozaki):
    rng = np.random.default_rng(3 * n + nrhs)
    A = spd(rng, n)
    factored, blocks, info = potrf_inv(ctx, A, n)
    assert info == 0
    L = np.tril(factored[:n, :n])
    ldb = n + 5
    B = np.full((max(nrhs, 1), ldb), 555.0)
    B[:nrhs, :n] = rng.standard_normal((nrhs, n))
    dL, dLinv, dB = ctx.to_device(L), ctx.to_device(blocks), ctx.to_device(B)
    with ctx.options(ozaki=ozaki):
        ctx._check(ctx.lib.b2gp_trsm_inv(ctx.h, n, nrhs, dL.ptr, n, dLinv.ptr, dB.ptr, ldb))
    got = dB.download()
    assert (got[:, n:] == 555.0).all() and (got[nrhs:] == B[nrhs:]).all(), "wrote outside the nrhs x n block"
    if nrhs:
        ref = sla.solve_triangular(L, B[:nrhs, :n].T, lower=True).T          # B L^{-T}
        assert_close(got[:nrhs, :n], ref, 1e-11 if ozaki == 0 else 1e-10, f"B L^-T, n={n} nrhs={nrhs} ozaki={ozaki}")


def rowdot(ctx, R, w, scale, dot0, nrm0, accumulate, rows=None, length=None):
    rows = R.shape[0] if rows is None else rows
    length = R.shape[1] - 3 if length is None else length          # ldr = len + 3
    dR, dw = ctx.to_device(R), (None if w is None else ctx.to_device(w))
    ddot = None if dot0 is None else ctx.to_device(dot0)
    dnrm = None if nrm0 is None else ctx.to_device(nrm0)
    ctx._check(ctx.lib.b2gp_rowdot(ctx.h, rows, length, dR.ptr, R.shape[1], None if dw is None else dw.ptr, float(scale),
                                   None if ddot is None else ddot.ptr, None if dnrm is None else dnrm.ptr, int(accumulate)))
    return (None if ddot is None else ddot.download()), (None if dnrm is None else dnrm.download())


@pytest.mark.parametrize("accumulate", [0, 1])
def test_rowdot(ctx, accumulate):
    rng = np.random.default_rng(9)
    rows, length = 37, 300
    R = rng.standard_normal((rows, length + 3))
    R[:, length:] = 1e300                                 # beyond len: must not be read
    w = rng.standard_normal(length)
    dot0, nrm0 = rng.standard_normal(rows), rng.standard_normal(rows)
    base_d, base_n = (dot0, nrm0) if accumulate else (0.0, 0.0)
    rd = base_d + 0.75 * (R[:, :length] @ w)
    rn = base_n + (R[:, :length] ** 2).sum(1)
    dot, nrm = rowdot(ctx, R, w, 0.75, dot0, nrm0, accumulate)
    assert_close(dot, rd, 1e-13, "dot")
    assert_close(nrm, rn, 1e-13, "nrm")
    dot, nrm = rowdot(ctx, R, None, 0.75, None, nrm0, accumulate)            # dot NULL (and w NULL)
    assert dot is None
    assert_close(nrm, rn, 1e-13, "nrm alone")
    dot, nrm = rowdot(ctx, R, w, 0.75, dot0, None, accumulate)               # nrm NULL
    assert_close(dot, rd, 1e-13, "dot alone")
    dot, nrm = rowdot(ctx, R, w, 0.75, dot0, nrm0, accumulate, rows=0)      # no rows: nothing written
    assert np.array_equal(dot, dot0) and np.array_equal(nrm, nrm0)
    dot, nrm = rowdot(ctx, R, w, 0.75, dot0, nrm0, accumulate, length=0)    # empty rows: the sums are 0
    assert np.array_equal(dot, dot0 if accumulate else np.zeros(rows)) and np.array_equal(nrm, nrm0 if accumulate else np.zeros(rows))


def test_copy2d_strided(ctx):
    rng = np.random.default_rng(10)
    src = rng.standard_normal((50, 77))
    dst0 = np.full((60, 91), 3.5)
    for rows, cols in [(50, 70), (1, 1), (0, 70), (50, 0)]:
        dsrc, ddst = ctx.to_device(src), ctx.to_device(dst0)
        ctx._check(ctx.lib.b2gp_copy2d(ctx.h, ddst.ptr, 91, dsrc.ptr, 77, rows, cols))
        ref = dst0.copy()
        ref[:rows, :cols] = src[:rows, :cols]
        assert np.array_equal(ddst.download(), ref), (rows, cols)


# ------------------------------------------------------------------ 4b. GpuOps and the NumPy stand-in agree
def test_gpu_ops_match_the_numpy_stand_in():
    torch = pytest.importorskip("torch")
    from dist_helpers import NumpyOps
    from gpax_b200.distributed import GpuOps
    gops, nops = GpuOps(device=0), NumpyOps()
    rng = np.random.default_rng(12)

    def both(fn, *arrays):
        """fn(ops, *tensors) on each implementation with the same inputs; returns the arrays afterwards and fn's values"""
        out = []
        for ops in (gops, nops):
            ts = [None if a is None else ops.from_numpy(a.copy()) for a in arrays]     # the stand-in shares memory
            v = fn(ops, *ts)
            ops.sync()
            out.append(([None if t is None else ops.to_numpy(t) for t in ts], v))
        return out

    n = 300
    A = spd(rng, n)
    nb_lin = 3 * 128 * 128
    (ga, gi), (na, ni) = both(lambda o, a, l: o.potrf_inv(a, l), A, np.zeros(nb_lin))
    assert gi == ni == 0
    assert_close(np.tril(ga[0]), np.tril(na[0]), 1e-12, "potrf_inv L")
    g_bl, n_bl = ga[1].reshape(3, 128, 128), na[1].reshape(3, 128, 128)
    for b, w in enumerate((128, 128, 44)):
        assert_close(g_bl[b, :w, :w], n_bl[b, :w, :w], 1e-11, f"potrf_inv block {b}")
    for j in (0, 150):
        bad = A.copy()
        bad[j, j] -= np.linalg.cholesky(A)[j, j] ** 2 + 1.0
        (_, gi), (_, ni) = both(lambda o, a, l: o.potrf_inv(a, l), bad, np.zeros(nb_lin))
        assert gi == ni == j + 1, (gi, ni)
    L, linv = np.tril(ga[0]), ga[1]
    for nrhs in (1, 1100):
        B = rng.standard_normal((nrhs, n))
        (g, _), (nn, _) = both(lambda o, l, li, b: o.trsm_inv(l, li, b), L, linv, B)
        assert_close(g[2], nn[2], 1e-11, f"trsm_inv nrhs={nrhs}")
    R, w = rng.standard_normal((40, 200)), rng.standard_normal(200)
    for acc in (0, 1):
        d0, n0 = rng.standard_normal(40), rng.standard_normal(40)
        (g, _), (nn, _) = both(lambda o, r, ww, d, q: o.rowdot(r, ww, d, q, acc), R, w, d0, n0)
        assert_close(g[2], nn[2], 1e-13, "rowdot dot")
        assert_close(g[3], nn[3], 1e-13, "rowdot nrm")
        (g, _), (nn, _) = both(lambda o, r, q: o.rowdot(r, None, None, q, acc), R, n0)
        assert_close(g[1], nn[1], 1e-13, "rowdot nrm only")
    (g, _), (nn, _) = both(lambda o, dst, src: o.copy(dst[3:20, 5:60], src[:17, 10:65]), np.zeros((30, 70)), R)
    assert np.array_equal(g[0], nn[0])
    N, M, P = 800, 96, 40
    X, y, Xu, Xn, theta = sparse_problem(N, M, P, 2, "Matern")
    (g, gi), (nn, ni) = both(lambda o, xu, x, yy, K, c: o.sparse_partial("Matern", xu, x, yy, theta, 1e-5, K, c),
                             Xu, X, y, np.zeros((M, M)), np.zeros(M))
    assert gi == ni == 0
    scale = np.abs(nn[3]).max()
    assert_close(np.tril(g[3]), nn[3], 1e-9, "sparse_partial Kpart")
    assert_close(g[4], nn[4], 1e-9 * max(1.0, scale / np.abs(nn[4]).max()), "sparse_partial cpart")
    Ks, cs = nn[3], nn[4]
    for noiseless in (False, True):
        (g, gi), (nn, ni) = both(lambda o, xu, K, c, xn, m, v, cv: o.sparse_finish("Matern", xu, K, c, xn, theta, noiseless, 1e-5, m, v, cv),
                                 Xu, Ks, cs, Xn, np.zeros(P), np.zeros(P), np.zeros((P, P)))
        assert gi == ni == 0
        for k, name in ((4, "mean"), (5, "var"), (6, "cov")):
            assert_close(g[k], nn[k], 1e-8, f"sparse_finish {name} noiseless={noiseless}")
    for kw, sign in (({"k_scale": -1.0}, 1), ({"noise": -0.05}, -1)):
        X, y, Xu, Xn, th = sparse_problem(N, M, P, 2, "RBF", **kw)
        (g, gi), (nn, ni) = both(lambda o, xu, x, yy, K, c: o.sparse_partial("RBF", xu, x, yy, th, 1e-5, K, c),
                                 Xu, X, y, np.zeros((M, M)), np.zeros(M))
        assert (gi > 0) == (ni > 0) == (sign > 0) and (gi == ni if sign > 0 else gi == ni == 0)
        (g, gi), (nn, ni) = both(lambda o, xu, K, c, xn, m, v: o.sparse_finish("RBF", xu, K, c, xn, th, False, 1e-5, m, v, None),
                                 Xu, g[3] if sign < 0 else np.zeros((M, M)), g[4] if sign < 0 else np.zeros(M), Xn, np.zeros(P), np.zeros(P))
        assert gi == ni and np.sign(gi) == sign, (gi, ni)
        assert np.isnan(g[4]).all() and np.isnan(nn[4]).all()
