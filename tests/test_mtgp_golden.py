"""CPU: oracle/mtgp_oracle.py and the host model programs against reference_vectors_mt.npz -- the reference's own MultiTaskGP /
CoregGP get_mvn_posterior and model() executed by tests/golden/make_golden_mt.py."""
import os

import numpy as np
import pytest

from oracle import mtgp_oracle as mo

GOLDEN_MT = os.path.join(os.path.dirname(__file__), "golden", "reference_vectors_mt.npz")

# tag -> (kernel, shared input space, number of tasks)
POSTERIORS = {"mt_matern_nl0": ("Matern", False, 3), "mt_matern_nl1": ("Matern", False, 3), "kron_rbf": ("RBF", True, 2),
              "mt_periodic": ("Periodic", False, 3), "coreg_rbf": ("RBF", False, 3), "coreg_rbf_pn": ("RBF", False, 3)}
MODELS = {"model_mt_matern": ("Matern", False, 3), "model_mt_periodic": ("Periodic", False, 3), "model_kron_rbf": ("RBF", True, 2),
          "model_coreg_rbf": ("RBF", False, 3), "model_coreg_periodic": ("Periodic", False, 3)}


@pytest.fixture(scope="module")
def gm():
    return np.load(GOLDEN_MT)


def latent_form(p, coreg):
    """a golden parameter dict -> the oracle's latent form (CoregGP's parameters gain the latent axis of length 1)"""
    p = dict(p)
    p.setdefault("k_scale", np.ones(1) if coreg else np.ones(len(p["W"])))
    p.setdefault("period", None)
    if coreg:
        for k in ("k_length", "k_scale", "W", "v", "period"):
            if p[k] is not None:
                p[k] = np.asarray(p[k])[None]
    return p


def golden_params(gm, tag, prefix):
    return {k[len(tag) + len(prefix):]: gm[k] for k in gm.files if k.startswith(tag + prefix)}


@pytest.mark.parametrize("tag", sorted(POSTERIORS))
def test_oracle_posterior_matches_the_reference(gm, tag):
    kind, shared, T = POSTERIORS[tag]
    p = latent_form(golden_params(gm, tag, "_p_"), tag.startswith("coreg"))
    mean, cov = mo.posterior(gm[tag + "_X"], gm[tag + "_y"], gm[tag + "_Xnew"], p, kind, shared, T, noiseless=tag.endswith("nl1"))
    np.testing.assert_allclose(mean, gm[tag + "_mean"], rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(cov, gm[tag + "_cov"], rtol=1e-9, atol=1e-10)


@pytest.mark.parametrize("tag", sorted(MODELS))
def test_oracle_covariance_of_the_y_site(gm, tag):
    """the fit-side covariance, noise and jitter included once per latent"""
    kind, shared, T = MODELS[tag]
    p = latent_form(golden_params(gm, tag, "_v_"), "coreg" in tag)
    K = mo.lcm_cov(gm[tag + "_X"], gm[tag + "_X"], p, p["noise"], kind, shared, T)
    np.testing.assert_allclose(K, gm[tag + "_ycov"], rtol=1e-13)


def test_host_programs_record_the_reference_sites(gm):
    from gpax_b200 import CoregGP, MultiTaskGP
    from gpax_b200 import priors as P
    models = {"model_mt_matern": (MultiTaskGP(1, "Matern", num_latents=2, rank=2), (3, 2, 2)),
              "model_mt_periodic": (MultiTaskGP(1, "Periodic", num_latents=2, rank=2), (3, 2, 2)),
              "model_kron_rbf": (MultiTaskGP(2, "RBF", num_latents=2, shared_input_space=True, num_tasks=2, output_scale=True), (2, 1, 2)),
              "model_coreg_rbf": (CoregGP(1, "RBF"), (3, 1, 1)),
              "model_coreg_periodic": (CoregGP(1, "Periodic"), (3, 1, 1))}
    for tag, (m, (T, R, L)) in models.items():
        m.X_train = gm[tag + "_X"]
        _, sites, det = P.run_program(lambda: m._model_program(T, R, L))
        shapes = [",".join(map(str, s.shape)) for s in sites.values()]
        assert list(sites) == list(gm[tag + "_site_names"]), tag
        assert shapes == list(gm[tag + "_site_shapes"]), tag
        assert list(det) == list(gm[tag + "_det_names"]), tag
