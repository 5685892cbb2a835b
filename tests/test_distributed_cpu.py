"""CPU, gloo, world_size 2: host logic of the multi-rank paths (gpax_b200/distributed.py) with the NumPy ops
stand-in from tests/dist_helpers.py, checked against the oracle."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import oracle


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, cases, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        for case in cases:
            _one_case(rank, world, case, q)
    finally:
        dist.destroy_process_group()


def _one_case(rank, world, case, q):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from dist_helpers import NumpyOps
    from gpax_b200.distributed import BlockCyclicGP, sharded_sparse_posterior
    ops = NumpyOps()
    rng = np.random.default_rng(11)
    if True:
        if case == "chol":
            N, P, d, nb = 700, 37, 2, 128       # 6 block columns, ragged last one, 3 per rank
            X = rng.uniform(0, 1, (N, d))
            y = np.sin(5 * X[:, 0]) + 0.1 * rng.standard_normal(N)
            Xn = rng.uniform(0, 1, (P, d))
            theta = np.array([0.3, 0.4, 1.1, 0.1, 1.0])
            gp = BlockCyclicGP(ops, N, nb)
            assert gp.owned == [j for j in range(6) if j % world == rank]
            mean, var, info = gp.posterior("Matern", ops.from_numpy(X), ops.from_numpy(y), ops.from_numpy(Xn), theta)
            q.put((rank, "chol", mean, var, info, gp.bytes_broadcast))
        elif case == "notpd":
            N, d, nb = 300, 1, 128
            X = rng.uniform(0, 1, (N, d))
            theta = np.array([0.3, -1.0, 0.1, 1.0])    # negative k_scale: indefinite K
            gp = BlockCyclicGP(ops, N, nb)
            mean, var, info = gp.posterior("RBF", ops.from_numpy(X), ops.from_numpy(rng.standard_normal(N)),
                                           ops.from_numpy(X[:5]), theta)
            q.put((rank, "notpd", mean, var, info, 0))
        else:
            N, M, P, d = 400, 48, 21, 2
            X = rng.uniform(0, 1, (N, d))
            y = np.sin(5 * X[:, 0]) + 0.1 * rng.standard_normal(N)
            Xu = X[rng.choice(N, M, replace=False)]
            Xn = rng.uniform(0, 1, (P, d))
            theta = np.array([0.4, 0.4, 1.0, 0.1, 1.0])
            lo, hi = rank * N // world, (rank + 1) * N // world
            out = sharded_sparse_posterior(ops, "RBF", ops.from_numpy(Xu), ops.from_numpy(X[lo:hi]), ops.from_numpy(y[lo:hi]),
                                           ops.from_numpy(Xn), theta, jitter=1e-5, want_cov=True)
            q.put((rank, "sparse", out["mean"], out["var"], out["info"], out["cov"]))


_CASES = ("chol", "notpd", "sparse")
_RESULTS = {}


def _run(case, world=2):
    """all cases run in ONE pair of spawned processes (importing torch in a fresh process is slow)"""
    if not _RESULTS:
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_worker, args=(r, world, port, _CASES, q)) for r in range(world)]
        for p in procs:
            p.start()
        res = [q.get(timeout=300) for _ in range(world * len(_CASES))]
        for p in procs:
            p.join(120)
            assert p.exitcode == 0
        for c in _CASES:
            _RESULTS[c] = sorted([t for t in res if t[1] == c], key=lambda t: t[0])
    return _RESULTS[case]


def test_block_cyclic_posterior_two_ranks():
    res = _run("chol")
    rng = np.random.default_rng(11)
    N, P, d = 700, 37, 2
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, d))
    params = {"k_length": np.array([0.3, 0.4]), "k_scale": 1.1, "noise": 0.1}
    ref_mean, ref_cov = oracle.exact_posterior(X, y, Xn, params, "Matern")
    for rank, _, mean, var, info, nbytes in res:
        assert info == 0
        np.testing.assert_allclose(mean, ref_mean, rtol=1e-9, atol=1e-9 * np.abs(ref_mean).max())
        np.testing.assert_allclose(var, np.diag(ref_cov), rtol=1e-9, atol=1e-9 * np.abs(ref_cov).max())
        # every rank saw every panel: sum_k (N - k nb) * nb * 8 bytes
        assert nbytes == sum((N - k * 128) * 128 * 8 for k in range(6))
    np.testing.assert_array_equal(res[0][2], res[1][2])      # replicated result identical on both ranks


def test_block_cyclic_not_positive_definite():
    for rank, _, mean, var, info, _ in _run("notpd"):
        assert info > 0 and np.isnan(mean).all() and np.isnan(var).all()


def test_sharded_sparse_two_ranks():
    res = _run("sparse")
    rng = np.random.default_rng(11)
    N, M, P, d = 400, 48, 21, 2
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(5 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.choice(N, M, replace=False)]
    Xn = rng.uniform(0, 1, (P, d))
    params = {"k_length": np.array([0.4, 0.4]), "k_scale": 1.0, "noise": 0.1}
    ref_mean, ref_cov = oracle.sparse_posterior(X, y, Xu, Xn, params, "RBF", jitter=1e-5)
    for rank, _, mean, var, info, cov in res:
        assert info == 0
        np.testing.assert_allclose(mean, ref_mean, rtol=1e-7, atol=1e-7 * np.abs(ref_mean).max())
        np.testing.assert_allclose(cov, ref_cov, rtol=1e-7, atol=1e-7 * np.abs(ref_cov).max())
        np.testing.assert_allclose(var, np.diag(ref_cov), rtol=1e-7, atol=1e-7 * np.abs(ref_cov).max())


def test_stand_in_potrf_inv_reports_the_first_bad_pivot_and_exports_the_block_inverses():
    """the stand-in's potrf_inv reports what b2gp_potrf_inv reports (BlockCyclicGP._panel turns it into k * nb + i)"""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from dist_helpers import NumpyOps
    ops = NumpyOps()
    rng = np.random.default_rng(4)
    n = 300
    G = rng.standard_normal((n, n))
    A = G @ G.T / n + np.eye(n)
    L = np.linalg.cholesky(A)
    a, linv = ops.from_numpy(A), ops.zeros((3 * 128 * 128,))
    assert ops.potrf_inv(a, linv) == 0
    np.testing.assert_allclose(np.tril(a.numpy()), L, rtol=1e-12, atol=1e-12)
    blocks = linv.numpy().reshape(3, 128, 128)
    for b, (lo, hi) in enumerate([(0, 128), (128, 256), (256, 300)]):
        np.testing.assert_allclose(blocks[b, :hi - lo, :hi - lo] @ L[lo:hi, lo:hi], np.eye(hi - lo), atol=1e-12)
    assert not blocks[2, 44:].any() and not blocks[2, :, 44:].any()
    for j in (0, 127, 200):
        bad = A.copy()
        bad[j, j] -= L[j, j] ** 2 + 1.0            # pivot j becomes sqrt(-1); pivots before it are untouched
        assert ops.potrf_inv(ops.from_numpy(bad), linv) == j + 1


def test_single_rank_degenerates_to_local(monkeypatch):
    """world_size 1 (no process group): no collective is issued"""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from dist_helpers import NumpyOps
    from gpax_b200.distributed import BlockCyclicGP
    ops = NumpyOps()
    rng = np.random.default_rng(2)
    N, P = 260, 9
    X = rng.uniform(0, 1, (N, 1))
    y = rng.standard_normal(N)
    Xn = rng.uniform(0, 1, (P, 1))
    theta = np.array([0.2, 1.0, 0.2, 1.0])
    gp = BlockCyclicGP(ops, N, 128)
    mean, var, info = gp.posterior("RBF", ops.from_numpy(X), ops.from_numpy(y), ops.from_numpy(Xn), theta)
    ref_mean, ref_cov = oracle.exact_posterior(X, y, Xn, {"k_length": np.array([0.2]), "k_scale": 1.0, "noise": 0.2}, "RBF")
    assert info == 0 and gp.bytes_broadcast == 0
    np.testing.assert_allclose(mean, ref_mean, rtol=1e-9, atol=1e-9 * np.abs(ref_mean).max())
    np.testing.assert_allclose(var, np.diag(ref_cov), rtol=1e-9, atol=1e-9 * np.abs(ref_cov).max())
