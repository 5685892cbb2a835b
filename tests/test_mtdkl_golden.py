"""The NumPy oracle of multi-task deep kernel learning (oracle/mtdkl_oracle.py) and viMTDKL's host program against the
golden vectors generated from the reference's own vi_mtdkl.py (tests/golden/make_golden_mtdkl.py): the posterior in both
forms with one and two latents, noiseless both ways, the prediction, the covariance model() gives the "y" site, and the
names and shapes of the kernel sites."""
import os

import numpy as np
import pytest

from oracle import dkl_oracle as dko
from oracle import mtdkl_oracle as mdo
from oracle import mtgp_oracle as mo

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_mtdkl.npz"))
NAMES = ["mlp/~/linear", "mlp/~/linear_1", "mlp/~/linear_2"]
TAGS = ["mt_L1", "mt_L2", "kron_L1", "kron_L2"]
T = 3


def case(tag):
    shared = tag.startswith("kron")
    layers = [(G[f"{tag}_{n}_w"], G[f"{tag}_{n}_b"]) for n in NAMES]
    p = {k: G[f"{tag}_p_{k}"] for k in ("k_length", "k_scale", "W", "v", "noise")}
    p["k_scale"] = p["k_scale"].reshape(-1)
    X, Xn = G[tag + "_X"], G[tag + "_X_new"]
    if shared:
        return shared, "RBF", X, None, Xn, None, layers, p
    return shared, "Matern", X[:, :-1], X[:, -1].astype(int), Xn[:, :-1], Xn[:, -1].astype(int), layers, p


def _close(got, ref, tol=1e-9):
    np.testing.assert_allclose(got, ref, rtol=tol, atol=tol * np.abs(ref).max())


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_posterior_and_predict(tag):
    shared, kind, X, tX, Xn, tN, layers, p = case(tag)
    for nl in (False, True):
        mean, cov = mdo.posterior(kind, X, tX, G[tag + "_y"], Xn, tN, layers, "relu", p, shared, T, nl)
        _close(mean, G[f"{tag}_mean_noiseless{int(nl)}"])
        _close(cov, G[f"{tag}_cov_noiseless{int(nl)}"])
        if not nl:
            _close(mean, G[tag + "_predict_mean"])
            _close(np.diag(cov), G[tag + "_predict_var"])


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_covariance_of_the_y_site(tag):
    shared, kind, X, tX, _, _, layers, p = case(tag)
    z = dko.mlp_forward(X, layers, "relu")[-1]
    Xg = z if shared else np.column_stack([z, tX])
    _close(mo.lcm_cov(Xg, Xg, p, p["noise"], kind, shared, T), G[tag + "_ycov"], 1e-12)


@pytest.mark.parametrize("tag", TAGS)
def test_host_program_records_the_reference_sites(tag):
    from gpax_b200 import viMTDKL
    shared = tag.startswith("kron")
    L = int(tag[-1])
    m = viMTDKL(6, 2, "RBF" if shared else "Matern", num_latents=L, shared_input_space=shared, num_tasks=T if shared else None,
                rank=2)
    m.X_train = G[tag + "_X"]
    sites = m._site_list()
    assert [n for n, _, _ in sites] == list(G[tag + "_site_names"])
    assert [",".join(map(str, sh)) for _, _, sh in sites] == list(G[tag + "_site_shapes"])
