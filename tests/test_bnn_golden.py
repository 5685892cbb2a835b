"""The NumPy oracle of BNN (oracle/bnn_oracle.py) and BNN's host-side layout against the golden vectors generated from the
reference's own bnn.py / spm.py (tests/golden/make_golden_bnn.py): get_mlp for the default and a custom hidden_dim with one
and three outputs, the prior program's sites and shapes, sample_single_posterior_predictive with injected normals, and
_set_data's shapes."""
import os

import numpy as np
import pytest

from oracle import bnn_oracle as bo

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_bnn.npz"))
CASES = [str(c) for c in G["cases"]]
HIDDEN = {"default": [64, 32], "custom": [16, 8, 4]}


def _close(got, ref, tol=1e-13):
    np.testing.assert_allclose(got, ref, rtol=tol, atol=tol * np.abs(ref).max())


def _case(case):
    tag, o = case.split("_")
    h, O = HIDDEN[tag], int(o[1:])
    L = len(h) + 1
    params = {f"{p}{i}": G[f"{case}_{p}{i}"] for i in range(L) for p in ("w", "b")}
    return h, O, params


def test_cases_cover_the_grid():
    assert sorted(CASES) == ["custom_O1", "custom_O3", "default_O1", "default_O3"]


@pytest.mark.parametrize("case", CASES)
def test_sites_and_flat_layout(case):
    from gpax_b200 import BNN
    h, O, params = _case(case)
    D = G["X_new"].shape[1]
    m = BNN(D, O, hidden_dim=None if case.startswith("default") else h)
    assert list(G[f"{case}_sites"]) == m.site_names()[:-1]
    for name, shape in zip(G[f"{case}_sites"], G[f"{case}_shapes"]):
        want = tuple(int(s) for s in shape if s)
        assert params[str(name)].shape == want
    flat = m.to_flat(params)
    back = m.from_flat(flat)
    assert all(np.array_equal(back[k], params[k]) for k in params)


@pytest.mark.parametrize("case", CASES)
def test_oracle_mlp_and_single_posterior_predictive(case):
    from gpax_b200 import BNN
    h, O, params = _case(case)
    Xn = G["X_new"]
    D = Xn.shape[1]
    flat = BNN(D, O, hidden_dim=h).to_flat(params)
    loc, ys = bo.predict(Xn, D, h + [O], flat, [0.17], G[f"{case}_eps"][None])
    _close(loc[0], G[f"{case}_mlp"])
    _close(loc[0], G[f"{case}_loc"])
    _close(ys[0], G[f"{case}_sample"])


def test_set_data_shapes():
    from gpax_b200 import BNN
    m = BNN(1, 1)
    x1, y1 = G["set_data_X1"], G["set_data_y1"]
    X, y = m._set_data(x1, y1)
    X2, y2 = BNN(2, 2)._set_data(np.ones((7, 2)), np.ones((7, 2)))
    got = [X.shape, y.shape, m._set_data(x1).shape, X2.shape, y2.shape]
    assert [tuple(s) for s in G["set_data_shapes"]] == got
