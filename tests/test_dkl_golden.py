"""The NumPy oracle of deep kernel learning (oracle/dkl_oracle.py) against the golden vectors generated from the reference's
own vidkl.py / dkl.py (tests/golden/make_golden_dkl.py): the MLP, the haiku naming and orientation, the posterior with and
without noise on k_pp, and the per-channel prediction."""
import os

import numpy as np
import pytest

from oracle import dkl_oracle as dko

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_dkl.npz"))
NAMES = ["mlp/~/linear", "mlp/~/linear_1", "mlp/~/linear_2"]
TOL = 1e-10


def _close(got, ref):
    np.testing.assert_allclose(got, ref, rtol=TOL, atol=TOL * np.abs(ref).max())


def dkl_case(tag):
    L = sum(1 for k in G.files if k.startswith(f"dkl_{tag}_w"))
    layers = [(G[f"dkl_{tag}_w{i}"], G[f"dkl_{tag}_b{i}"]) for i in range(L)]
    params = {"k_length": G[f"dkl_{tag}_k_length"], "k_scale": float(G[f"dkl_{tag}_k_scale"]),
              "noise": float(G[f"dkl_{tag}_noise"])}
    return layers, params


def vidkl_layers(prefix="vidkl", c=None):
    pick = (lambda a: a) if c is None else (lambda a: a[c])
    return [(pick(G[f"{prefix}_{n}_w"]), pick(G[f"{prefix}_{n}_b"])) for n in NAMES]


@pytest.mark.parametrize("tag", ["default", "custom"])
def test_dkl_posterior_and_embed(tag):
    layers, params = dkl_case(tag)
    mean, cov = dko.posterior("Matern", G["X"], G["y"], G["X_new"], layers, "tanh", params)
    _close(mean, G[f"dkl_{tag}_mean"])
    _close(cov, G[f"dkl_{tag}_cov"])
    for s, f in enumerate((1.0, 1.1)):
        z = dko.mlp_forward(G["X_new"], [(f * W, f * b) for W, b in layers], "tanh")[-1]
        _close(z, G[f"dkl_{tag}_embed"][s])


@pytest.mark.parametrize("noiseless", [False, True])
def test_vidkl_posterior(noiseless):
    kp = {"k_length": np.array([0.8, 1.1]), "k_scale": 1.3, "noise": 0.02}
    mean, cov = dko.posterior("RBF", G["X"], G["y"], G["X_new"], vidkl_layers(), "relu", kp, noiseless)
    _close(mean, G[f"vidkl_mean_noiseless{int(noiseless)}"])
    _close(cov, G[f"vidkl_cov_noiseless{int(noiseless)}"])
    if not noiseless:
        _close(mean, G["vidkl_predict_mean"])
        _close(np.diag(cov), G["vidkl_predict_var"])
    _close(dko.mlp_forward(G["X_new"], vidkl_layers(), "relu")[-1], G["vidkl_embed"])


def test_vidkl_three_channels():
    for c in range(3):
        kp = {"k_length": G["vidkl3_k_length"][c], "k_scale": float(G["vidkl3_k_scale"][c]), "noise": float(G["vidkl3_noise"][c])}
        mean, cov = dko.posterior("RBF", G["X"], G["vidkl3_Y"][c], G["X_new"], vidkl_layers("vidkl3", c), "relu", kp)
        _close(mean, G["vidkl3_predict_mean"][c])
        _close(np.diag(cov), G["vidkl3_predict_var"][c])
