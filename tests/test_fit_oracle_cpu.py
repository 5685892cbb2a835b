"""CPU: the references of tests/test_gpu_fit_paths.py are right, and its tolerance is tight enough to catch real defects.

1. fit_oracle.mll_grad / elbo_grad against the 60-digit arbiter (values in mpmath, gradients by mp.diff of them) to 1e-12
   relative to the size of the cancelling terms, for RBF, Matern and Periodic at d = 1, 3, 16, with the edges where the
   kernel formulas are delicate: duplicated rows under Matern (r = 0, where the 1e-12 under the square root acts), points
   exactly one period apart under Periodic, an inducing point on a training point.
2. the same against fp64 central differences on mid-size problems.
3. mutation checks: a named defect planted in the reference output (fit_oracle: `mutate=`) must fail the tolerance of the
   GPU case that stands for it.  A mutation that passed would mean that tolerance cannot see that bug."""
import numpy as np
import pytest

import test_gpu_fit_paths as gpu
from oracle import fit_oracle as fo

ARBITER = 1e-12


def _edges(kind, X, d):
    X = X.copy()
    if kind == "Matern":
        X[3] = X[1]                                        # duplicated row: r2 = 0
    if kind == "Periodic":
        X[5] = X[2]
        X[5, 0] += 0.7                                     # exactly one period (theta's period) apart along x_0
    return X


@pytest.mark.parametrize("d", [1, 3, 16])
@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
def test_mll_grad_matches_60_digits(kind, d):
    N = 10 if d == 16 else 16
    X, y, theta = fo.mll_problem(kind, N, d, 3 + d)
    X = _edges(kind, X, d)
    nv = np.linspace(1e-3, 0.3, N) if kind == "RBF" else None
    v, g, _, gnv, sc = fo.mll_grad(kind, X, y, theta, 1e-6, nv)
    vm, gm, gnvm = fo.mll_grad_mp(kind, X, y, theta, 1e-6, nv)
    assert abs(v - vm) <= ARBITER * abs(vm)
    assert np.all(np.abs(g - gm) <= ARBITER * (np.abs(gm) + sc)), (g - gm) / (np.abs(gm) + sc)
    if kind != "Periodic":
        assert g[d + 2] == 0.0
    if nv is not None:
        np.testing.assert_allclose(gnv, gnvm, rtol=0, atol=ARBITER * np.abs(gnvm).max())


@pytest.mark.parametrize("d", [1, 3, 16])
@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
def test_elbo_grad_matches_60_digits(kind, d):
    M, N = (3, 10) if d == 16 else (5, 16)
    Xu, X, y, theta = fo.elbo_problem(kind, M, N, d, 7 + d)
    X = _edges(kind, X, d)
    Xu[0] = X[0]                                           # an inducing point on a training point
    v, g, gx, sc, sx, _ = fo.elbo_grad(kind, Xu, X, y, theta, 1e-5)
    vm, gm, gxm = fo.elbo_grad_mp(kind, Xu, X, y, theta, 1e-5)
    assert abs(v - vm) <= ARBITER * abs(vm)
    assert np.all(np.abs(g - gm) <= ARBITER * (np.abs(gm) + sc)), (g - gm) / (np.abs(gm) + sc)
    assert np.all(np.abs(gx - gxm) <= ARBITER * (np.abs(gxm) + sx)), (gx - gxm) / (np.abs(gxm) + sx)


def test_elbo_clipped_branch_matches_60_digits():
    """Xu = X, points far apart, jitter < 0: T < 0, so the trace term and its gradient are 0"""
    X, y, theta = gpu.separated_problem("RBF", 6)
    v, g, gx, sc, sx, T = fo.elbo_grad("RBF", X, X, y, theta, -1e-4)
    assert T < 0
    vm, gm, gxm = fo.elbo_grad_mp("RBF", X, X, y, theta, -1e-4)
    assert abs(v - vm) <= ARBITER * abs(vm)
    assert np.all(np.abs(g - gm) <= ARBITER * (np.abs(gm) + sc))
    assert np.all(np.abs(gx - gxm) <= ARBITER * (np.abs(gxm) + sx))


@pytest.mark.parametrize("kind", ["RBF", "Matern", "Periodic"])
def test_references_against_fp64_central_differences(kind):
    """a second, independent check on mid-size problems: h = 1e-5 in log theta (and in Xu), error O(h^2) + O(eps / h)"""
    h, rtol = 1e-5, 1e-6
    X, y, theta = fo.mll_problem(kind, 200, 2, 5)
    _, g, _, _, sc = fo.mll_grad(kind, X, y, theta, 1e-6)
    for p in range(5):
        tp, tm = theta.copy(), theta.copy()
        tp[p] *= np.exp(h)
        tm[p] *= np.exp(-h)
        fd = (fo.mll_grad(kind, X, y, tp, 1e-6)[0] - fo.mll_grad(kind, X, y, tm, 1e-6)[0]) / (2 * h)
        assert abs(g[p] - fd) <= rtol * (abs(fd) + sc[p]), (p, g[p], fd)
    Xu, X, y, theta = fo.elbo_problem(kind, 30, 200, 2, 6)
    _, g, gx, sc, sx, _ = fo.elbo_grad(kind, Xu, X, y, theta, 1e-5)
    for p in range(5):
        tp, tm = theta.copy(), theta.copy()
        tp[p] *= np.exp(h)
        tm[p] *= np.exp(-h)
        fd = (fo.elbo_grad(kind, Xu, X, y, tp, 1e-5)[0] - fo.elbo_grad(kind, Xu, X, y, tm, 1e-5)[0]) / (2 * h)
        assert abs(g[p] - fd) <= rtol * (abs(fd) + sc[p]), (p, g[p], fd)
    for a, k in [(0, 0), (17, 1), (29, 0)]:
        Xp, Xm = Xu.copy(), Xu.copy()
        Xp[a, k] += h
        Xm[a, k] -= h
        fd = (fo.elbo_grad(kind, Xp, X, y, theta, 1e-5)[0] - fo.elbo_grad(kind, Xm, X, y, theta, 1e-5)[0]) / (2 * h)
        assert abs(gx[a, k] - fd) <= rtol * (abs(fd) + sx[a, k]), (a, k, gx[a, k], fd)


# ------------------------------------------------------------------ mutation checks
def _mll_case(name):
    """(kind, X, y, theta, planes) of the GPU case `name`"""
    if name == "kinv_syrk":
        return ("RBF",) + gpu.kinv_syrk_case() + (7,)
    return gpu.mll_default_case(int(name[len("default-N"):])) + (0,)


MLL_MUTATIONS = [("diag2", "default-N129"), ("diag2", "default-N1025"), ("drop_tile", "default-N65"),
                 ("drop_tile", "default-N129"), ("jitter_noise", "default-N257"), ("jitter_noise", "default-N1025"),
                 ("kinv_plane", "kinv_syrk")]


@pytest.mark.parametrize("mutation,case", MLL_MUTATIONS)
def test_mll_mutation_fails_the_gpu_tolerance(mutation, case):
    kind, X, y, theta, planes = _mll_case(case)
    t = fo.tau(fo.mll_cond(kind, X, theta, gpu.JITTER), planes)
    _, g, _, _, sc = fo.mll_grad(kind, X, y, theta, gpu.JITTER)
    _, gm, _, _, _ = fo.mll_grad(kind, X, y, theta, gpu.JITTER, mutate=mutation)
    assert fo.err_ratio(gm, g, sc, t) > 1.0, (mutation, case)


def _elbo_case(name):
    """(kind, Xu, X, y, theta, jitter) of the GPU case `name`"""
    if name.startswith("clip-"):
        kind, sign = name.split("-")[1:]
        X, y, theta = gpu.separated_problem(kind, 40)
        return kind, X, X, y, theta, (1e-5 if sign == "pos" else -1e-4)
    M, N, d = (int(v) for v in name.split("-")[1:])
    return gpu.elbo_default_case(M, N, d) + (1e-5,)


ELBO_MUTATIONS = [("clip", "clip-RBF-pos"), ("clip", "clip-RBF-neg"), ("clip", "clip-Matern-pos"), ("clip", "clip-Matern-neg"),
                  ("xu_kuu", "default-129-1001-3"), ("xu_kuu", "default-7-61-16"), ("xu_kuu", "default-300-300-3")]


@pytest.mark.parametrize("mutation,case", ELBO_MUTATIONS)
def test_elbo_mutation_fails_the_gpu_tolerance(mutation, case):
    kind, Xu, X, y, theta, jitter = _elbo_case(case)
    t = fo.tau(fo.kuu_cond(kind, Xu, theta, jitter), 0)
    _, g, gx, sc, sx, _ = fo.elbo_grad(kind, Xu, X, y, theta, jitter)
    _, gm, gxm, _, _, _ = fo.elbo_grad(kind, Xu, X, y, theta, jitter, mutate=mutation)
    assert max(fo.err_ratio(gm, g, sc, t), fo.err_ratio(gxm, gx, sx, t)) > 1.0, (mutation, case)
