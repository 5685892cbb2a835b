"""The NumPy oracle of iBNN / vi_iBNN (oracle/ibnn_oracle.py) against the golden vectors generated from the reference's own
ibnn.py / vi_ibnn.py (tests/golden/make_golden_ibnn.py): the NNGP Gram matrices, get_mvn_posterior and viGP.predict for
erf and ReLU, depths 1 and 3, d = 1 and 5, with and without noise on k_pp."""
import os

import numpy as np
import pytest

from oracle import ibnn_oracle as io

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_ibnn.npz"))
CASES = [str(c) for c in G["cases"]]
PARAMS = dict(zip(("var_b", "var_w", "noise"), G["params"]))


def _close(got, ref, tol):
    np.testing.assert_allclose(got, ref, rtol=tol, atol=tol * np.abs(ref).max())


def _case(tag):
    d, act, depth = tag.split("_")
    return G[d + "_X"], G[d + "_y"], G[d + "_Xnew"], act, int(depth[1:])


def test_cases_cover_the_grid():
    assert len(CASES) == 8
    assert {c.split("_")[0] for c in CASES} == {"d1", "d5"} and {c.split("_")[1] for c in CASES} == {"erf", "relu"}


@pytest.mark.parametrize("tag", CASES)
def test_kernel(tag):
    X, _, Xn, act, depth = _case(tag)
    _close(io.kernel(X, X, PARAMS, PARAMS["noise"], 1e-6, act, depth), G[tag + "_Kxx"], 1e-12)
    _close(io.kernel(Xn, X, PARAMS, 0.0, 0.0, act, depth), G[tag + "_Kpx"], 1e-12)


@pytest.mark.parametrize("noiseless", [False, True])
@pytest.mark.parametrize("tag", CASES)
def test_posterior_and_vi_predict(tag, noiseless):
    X, y, Xn, act, depth = _case(tag)
    key = f"{tag}_nl{int(noiseless)}"
    mean, cov = io.posterior(X, y, Xn, PARAMS, act, depth, noiseless)
    _close(mean, G[key + "_mean"], 1e-9)
    _close(cov, G[key + "_cov"], 1e-9)
    vm, vv = io.vi_predict(X, y, Xn, PARAMS, act, depth, noiseless)
    _close(vm, G[key + "_vimean"], 1e-9)
    _close(vv, G[key + "_vivar"], 1e-9)
