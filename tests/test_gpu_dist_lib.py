"""GPU: the in-library multi-GPU posterior (b2gp_dist_posterior, gpax_b200/csrc/dist.cuh) against the single-GPU posterior.
A 1 x 1 "grid" runs the whole block-cyclic machinery (tile lists, row maps, look-ahead order) on one GPU; with two or more
GPUs visible the same problem runs as one process per GPU over NCCL on 1 x 2, 2 x 1 (and 2 x 2 / 2 x 4) grids."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import ROOT, assert_close
import oracle
from dist_lib_worker import SPARSE_SHAPE, problem
from dist_single_worker import sparse_problem

pytestmark = pytest.mark.gpu


def n_gpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return len([l for l in out.splitlines() if l.startswith("GPU ")])
    except Exception:  # noqa: BLE001
        return 0


def run_grid(pr, pc, N, P, nb, kernel, ozaki=-1, sparse=False):
    """ozaki=None: the workers set no option at all (the library's defaults).  sparse: the ranks also run the sharded sparse
    posterior.  Every worker is killed and reaped before this returns, also after a timeout or when one rank fails while
    the others wait in a collective."""
    world = pr * pc
    port = 29600 + (os.getpid() + 7 * pr + 13 * pc + N) % 300
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "res")
        procs = []
        try:
            for r in range(world):
                env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
                env.pop("B200GP_TEST_OZAKI", None)
                if ozaki is not None:
                    env["B200GP_TEST_OZAKI"] = str(ozaki)
                procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "dist_lib_worker.py"), str(pr), str(pc), str(N),
                                               str(P), str(nb), kernel, out] + (["sparse"] if sparse else []),
                                              env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
            logs = [p.communicate(timeout=600)[0] for p in procs]
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                p.communicate()
        for p, lg in zip(procs, logs):
            assert p.returncode == 0, lg[-3000:]
        return [dict(np.load(out + f".rank{r}.npz")) for r in range(world)]


def single_gpu(N, P, kernel, ozaki=-1):
    import gpax_b200
    X, y, Xn, theta = problem(N, P, kernel)
    ctx = gpax_b200.default_context()
    with ctx.options(ozaki=ozaki):
        return ctx.posterior(kernel, X, y, Xn, theta[None], want=("mean", "var"))


# The block-cyclic path runs EVERY update through the int8 kernel at k = nb, the single-GPU path only the large ones, so
# the two differ by the digit-plane arithmetic: ~1e-12 of the result's scale with 7 planes (54-bit operands), ~1e-10
# with the 6 planes the accuracy rule picks for this conditioning -- both far inside the 1e-9 parity bar.
TOL = {7: 2e-12, -1: 1e-9}


@pytest.mark.parametrize("N,P,nb,kernel", [(2048, 300, 256, "Matern"), (3072, 100, 512, "RBF"), (1024, 700, 128, "Periodic")])
def test_one_rank_grid_matches_single_gpu(N, P, nb, kernel):
    for oz in (7, -1):
        ref = single_gpu(N, P, kernel, oz)
        res = run_grid(1, 1, N, P, nb, kernel, oz)[0]
        assert res["info"] == 0
        em = np.abs(res["mean"] - ref["mean"][0]).max() / np.abs(ref["mean"][0]).max()
        ev = np.abs(res["var"] - ref["var"][0]).max() / np.abs(ref["var"][0]).max()
        print(f"1 x 1 grid N={N} nb={nb} {kernel} ozaki={oz}: scaled deviation from the single-GPU path mean {em:.1e} var {ev:.1e}")
        assert_close(res["mean"], ref["mean"][0], TOL[oz], f"mean, 1 x 1 grid, ozaki={oz}")
        assert_close(res["var"], ref["var"][0], TOL[oz], f"var, 1 x 1 grid, ozaki={oz}")


@pytest.mark.parametrize("pr,pc", [(1, 2), (2, 1), (2, 2), (2, 4)])
def test_process_grid_matches_single_gpu(pr, pc):
    if n_gpus() < pr * pc:
        pytest.skip(f"needs {pr * pc} GPUs")
    N, P, nb, kernel = 4096, 600, 256, "Matern"
    ref = single_gpu(N, P, kernel, 7)
    res = run_grid(pr, pc, N, P, nb, kernel, 7, sparse=True)
    one = run_grid(1, 1, N, P, nb, kernel, 7)[0] if (pr, pc) == (1, 2) else None
    for r in res:
        assert r["info"] == 0
        assert_close(r["mean"], ref["mean"][0], TOL[7], f"mean, {pr} x {pc} grid")     # SURVEY 8e: equal to the 1-GPU result to 1e-12
        assert_close(r["var"], ref["var"][0], TOL[7], f"var, {pr} x {pc} grid")
        np.testing.assert_array_equal(r["mean"], res[0]["mean"])                       # every rank holds the same result
    # the sharded sparse posterior: each rank's shard, the statistics summed by the in-library all-reduce
    Ns, M, Ps, ks = SPARSE_SHAPE
    X, y, Xu, Xn, theta = sparse_problem(Ns, M, Ps, 2, ks)
    params = {"k_length": theta[:2], "k_scale": theta[2], "noise": theta[3], "period": theta[4]}
    rmean, rcov = oracle.sparse_posterior(X, y, Xu, Xn, params, ks, jitter=1e-5)
    w = np.linalg.eigvalsh(oracle.get_kernel(ks)(Xu, Xu, params, jitter=1e-5))
    tol = 1e-9 * max(1.0, w[-1] / w[0] / 1e5)
    for r in res:
        assert r["sparse_info"] == 0
        assert_close(r["sparse_mean"], rmean, tol, f"sharded sparse mean, {pr * pc} ranks")
        assert_close(r["sparse_var"], np.diag(rcov), tol, f"sharded sparse var, {pr * pc} ranks")
        np.testing.assert_array_equal(r["sparse_mean"], res[0]["sparse_mean"])
        np.testing.assert_array_equal(r["sparse_var"], res[0]["sparse_var"])
    if one is not None:    # the same tiles and the same arithmetic on one GPU: only the order of the final reduction differs
        assert_close(res[0]["mean"], one["mean"], 1e-13, "1 x 2 grid vs 1 x 1 grid")
