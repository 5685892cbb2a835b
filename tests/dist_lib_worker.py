"""Worker of tests/test_gpu_dist_lib.py: one rank of the in-library multi-GPU posterior (env: RANK, WORLD_SIZE, LOCAL_RANK,
MASTER_ADDR, MASTER_PORT; argv: pr pc N P nb kernel outfile [sparse]).  With the optional last argument "sparse" the rank
also runs the N-sharded sparse posterior (b2gp_dist_sparse_posterior) on its shard of SPARSE_SHAPE."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def problem(N, P, kernel):
    rng = np.random.default_rng(77)
    d = 2
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    theta = np.array([0.25, 0.35, 1.1, 0.05, 0.9])
    return X, y, Xn, theta


SPARSE_SHAPE = (3000, 200, 150, "Matern")     # N, M, P, kernel of the sharded sparse case


def shard(N, rank, world):
    """rank's share [lo, hi) of N training points; uneven when world does not divide N"""
    return rank * N // world, (rank + 1) * N // world


def main():
    pr, pc, N, P, nb = (int(a) for a in sys.argv[1:6])
    kernel, out = sys.argv[6], sys.argv[7]
    from gpax_b200 import dist
    dc = dist.DistContext(grid=(pr, pc))
    if "B200GP_TEST_OZAKI" in os.environ:       # unset: the context keeps the library's defaults, as a user's would
        dc.ctx.set_option("ozaki", int(os.environ["B200GP_TEST_OZAKI"]))
    X, y, Xn, theta = problem(N, P, kernel)
    res = dc.posterior(kernel, X, y, Xn, theta, nb=nb)
    res2 = dc.posterior(kernel, X, y, Xn, theta, nb=nb)          # a second call reuses the cached lists / buffers
    assert np.array_equal(res["mean"], res2["mean"]) and np.array_equal(res["var"], res2["var"])
    np.savez(out + f".rank{dc.rank}.npz", mean=res["mean"], var=res["var"], info=res["info"], potrf_ms=res["timing"]["potrf_ms"],
             ozaki=dc.ctx.get_option("ozaki"), **(sparse(dc) if sys.argv[8:] == ["sparse"] else {}))
    dc.close()


def sparse(dc):
    from dist_single_worker import sparse_problem
    N, M, P, kernel = SPARSE_SHAPE
    X, y, Xu, Xn, theta = sparse_problem(N, M, P, 2, kernel)
    lo, hi = shard(N, dc.rank, dc.world)
    res = dc.sparse_posterior(kernel, Xu, X[lo:hi], y[lo:hi], Xn, theta, jitter=1e-5)
    return {"sparse_mean": res["mean"], "sparse_var": res["var"], "sparse_info": res["info"]}


if __name__ == "__main__":
    main()
