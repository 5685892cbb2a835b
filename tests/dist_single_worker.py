"""Worker of tests/test_gpu_dist_single.py: the collective entry points (b2gp_dist_posterior, b2gp_dist_sparse_posterior)
on a 1 x 1 process grid, many cases through ONE DistContext in ONE process (NCCL starts once).

argv: cases.json outdir.  cases.json is a list of dicts with an "id" and an "op" ("dense", "sparse" or "refuse"); the
result of each case is written to outdir/<id>.npz, in list order.  The problems are generated here and in the test from
the same functions, so only results travel."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SENTINEL = -12345.5          # var is pre-filled with this; a mean-only call must leave it untouched
DENSE_THETA = np.array([0.25, 0.35, 1.1, 0.05, 0.9])


def dense_problem(N, P, kernel, noise=0.05):
    """training points in the unit square; test points also outside it, so that some variances are O(k_scale)"""
    rng = np.random.default_rng(1000 + N + 7 * P)
    X = rng.uniform(0, 1, (N, 2))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(-0.3, 1.3, (P, 2))
    theta = DENSE_THETA.copy()
    theta[3] = noise
    return X, y, Xn, theta


def sparse_problem(N, M, P, d, kernel, k_scale=1.0, noise=0.05):
    rng = np.random.default_rng(2000 + N + 3 * M + P)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(9 * X[:, 0]) * np.cos(7 * X[:, -1]) + 0.05 * rng.standard_normal(N)
    Xu = X[rng.choice(N, M, replace=False)]
    Xn = rng.uniform(-0.2, 1.2, (P, d))
    theta = np.concatenate([np.full(d, 0.2), [k_scale, noise, 0.8]])
    return X, y, Xu, Xn, theta


def c5_problem():
    """bench.py's c5 workload (viSparseGP Matern, N = 262144, d = 2, M = 4096, P = 4096), generated the same way"""
    N, d, M, P = 262144, 2, 4096, 4096
    rng = np.random.default_rng(6)
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(9 * X[:, 0]) * np.cos(7 * X[:, 1]) + 0.05 * rng.standard_normal(N)
    Xu = X[rng.choice(N, M, replace=False)]
    Xn = rng.uniform(0, 1, (P, d))
    theta = np.array([0.2, 0.2, 1.0, 0.05, 1.0])
    return X, y, Xu, Xn, theta


def _opts(case):
    o = {}
    if case.get("ozaki") is not None:
        o["ozaki"] = case["ozaki"]
    if case.get("oz_cluster") is not None:
        o["oz_cluster"] = case["oz_cluster"]
    return o


def dense(dc, case):
    from gpax_b200 import _ffi
    X, y, Xn, theta = dense_problem(case["N"], case["P"], case["kernel"], case.get("noise", 0.05))
    P = Xn.shape[0]
    mean, var = np.full(P, SENTINEL), np.full(P, SENTINEL)
    info = C.c_int(0)
    flags = _ffi.OUT_MEAN | (_ffi.OUT_VAR if case.get("want_var", True) else 0)
    with dc.ctx.options(**_opts(case)):
        dc.ctx._check(dc.ctx.lib.b2gp_dist_posterior(
            dc.ctx.h, _ffi.KIND[case["kernel"]], _ffi._ptr(X), X.shape[0], _ffi._ptr(y), _ffi._ptr(Xn), P, 2, _ffi._ptr(theta),
            int(case.get("noiseless", False)), 1e-6, case["nb"], flags, _ffi._ptr(mean), _ffi._ptr(var), C.byref(info), None))
    return {"mean": mean, "var": var, "info": info.value}


def sparse(dc, case):
    from gpax_b200 import _ffi
    if case.get("c5"):
        X, y, Xu, Xn, theta = c5_problem()
    else:
        X, y, Xu, Xn, theta = sparse_problem(case["N"], case["M"], case["P"], case.get("d", 2), case["kernel"],
                                             case.get("k_scale", 1.0), case.get("noise", 0.05))
    M, d = Xu.shape
    P = Xn.shape[0]
    mean, var = np.full(P, SENTINEL), np.full(P, SENTINEL)
    info = C.c_int(0)
    flags = _ffi.OUT_MEAN | (_ffi.OUT_VAR if case.get("want_var", True) else 0)
    out = {}
    with dc.ctx.options(**_opts(case)):
        dc.ctx._check(dc.ctx.lib.b2gp_dist_sparse_posterior(
            dc.ctx.h, _ffi.KIND[case["kernel"]], _ffi._ptr(Xu), M, _ffi._ptr(X), X.shape[0], _ffi._ptr(y), _ffi._ptr(Xn), P, d,
            _ffi._ptr(theta), int(case.get("noiseless", False)), 1e-5, flags, _ffi._ptr(mean), _ffi._ptr(var), C.byref(info), None))
        if case.get("bits"):      # the single-GPU entry point on the same context, under the same options
            one = dc.ctx.sparse_posterior(case["kernel"], Xu, X, y, Xn, theta, noiseless=case.get("noiseless", False), jitter=1e-5,
                                          want=("mean", "var"))
            out.update(one_mean=one["mean"], one_var=one["var"], one_info=one["info"])
    out.update(mean=mean, var=var, info=info.value)
    return out


def refuse(dc, case):
    """one call with a bad argument: the library's return code and message (nothing may be written)"""
    from gpax_b200 import _ffi
    N, P, d = case.get("N", 256), 10, case.get("d", 2)
    rng = np.random.default_rng(5)
    X, y, Xn = rng.uniform(0, 1, (N, d)), rng.standard_normal(N), rng.uniform(0, 1, (P, d))
    theta = np.concatenate([np.full(d, 0.3), [1.0, 0.1, 1.0]])
    mean, var = np.full(P, SENTINEL), np.full(P, SENTINEL)
    info = C.c_int(7)
    kind = case.get("kind", 0)
    flags = case.get("flags", _ffi.OUT_MEAN | _ffi.OUT_VAR)
    lib = dc.ctx.lib
    if case["entry"] == "dense":
        rc = lib.b2gp_dist_posterior(dc.ctx.h, kind, _ffi._ptr(X), N, _ffi._ptr(y), _ffi._ptr(Xn), P, d, _ffi._ptr(theta), 0, 1e-6,
                                     case.get("nb", 128), flags, _ffi._ptr(mean), _ffi._ptr(var), C.byref(info), None)
    else:
        rc = lib.b2gp_dist_sparse_posterior(dc.ctx.h, kind, _ffi._ptr(X[:32]), 32, _ffi._ptr(X), N, _ffi._ptr(y), _ffi._ptr(Xn), P, d,
                                            _ffi._ptr(theta), 0, 1e-5, flags, _ffi._ptr(mean), _ffi._ptr(var), C.byref(info), None)
    msg = lib.b2gp_last_error(dc.ctx.h)
    return {"rc": rc, "msg": np.array(msg.decode() if msg else ""), "mean": mean, "var": var, "info": info.value}


def main():
    cases_file, outdir = sys.argv[1], sys.argv[2]
    with open(cases_file) as f:
        cases = json.load(f)
    from gpax_b200 import dist
    dc = dist.DistContext(grid=(1, 1), rank=0, world=1)
    try:
        for case in cases:
            res = {"dense": dense, "sparse": sparse, "refuse": refuse}[case["op"]](dc, case)
            np.savez(os.path.join(outdir, case["id"] + ".npz"), **res)
    finally:
        dc.close()


if __name__ == "__main__":
    main()
