"""
acquisition.py -- acquisition functions with the reference's surface: EI / UCB / POI / UE / KG / Thompson
(gpax/acquisition/acquisition.py:50-524 over base_acq.py:20-232), the q-batch forms qEI / qUCB / qPOI / qKG
(gpax/acquisition/batch_acquisition.py:60-282) and optimize_acq over a continuous box (gpax/acquisition/optimize.py).  The arithmetic runs on the GPU as epilogues of the posterior
(b2gp_acq_moments / b2gp_acq_samples / b2gp_kg, gpax_b200/csrc/acq.cuh); the penalties of
gpax/acquisition/penalties.py are O(P * recent) host arithmetic and stay on the host, as in the reference.
"""
import contextlib
from typing import Optional

import numpy as np

from . import prng
from .utils import posterior_eps

__all__ = ["EI", "UCB", "POI", "UE", "KG", "Thompson", "qEI", "qUCB", "qPOI", "qKG", "optimize_acq", "ei", "ucb", "poi", "ue",
           "compute_penalty"]


# ------------------------------------------------------------------ base functions on moments (base_acq.py:20-155)
def _ctx(model=None):
    from . import _ffi
    return model.ctx if model is not None else _ffi.default_context()


def ei(moments, best_f=None, maximize=False, ctx=None, **kwargs):
    mean, var = moments
    return (ctx or _ctx()).acq_moments("EI", mean, var, best_f, 0.0, maximize)


def ucb(moments, beta=0.25, maximize=False, ctx=None, **kwargs):
    mean, var = moments
    return (ctx or _ctx()).acq_moments("UCB", mean, var, None, beta, maximize)


def ue(moments, ctx=None, **kwargs):
    mean, var = moments
    return (ctx or _ctx()).acq_moments("UE", mean, var)


def poi(moments, best_f=None, xi=0.01, maximize=False, ctx=None, **kwargs):
    mean, var = moments
    return (ctx or _ctx()).acq_moments("POI", mean, var, best_f, xi, maximize)


# ------------------------------------------------------------------ penalties (penalties.py)
def _penalty_point(x, recent_points):
    if recent_points.ndim == 1:
        recent_points = recent_points[:, None]
    distances = np.linalg.norm(recent_points - x, axis=1)
    timestamps = 1 if len(recent_points) == 1 else np.arange(len(recent_points) + 1, 1, -1)
    return np.sum(1 / (distances + 1) / timestamps)


def compute_penalty(X, recent_points, penalty_type="delta", penalty_factor=1.0):
    """gpax/acquisition/penalties.py:15-45."""
    X, recent_points = np.asarray(X), np.asarray(recent_points)
    if penalty_type not in ["delta", "inverse_distance", "inverse distance"]:
        raise NotImplementedError("Avaialble penalty types are 'delta' and 'inverse distance'")
    if penalty_type == "delta":
        out = np.zeros(len(X))
        for single_point in recent_points:
            idx = np.where(np.all(X == single_point, axis=1))[0]
            if idx.size > 0:
                out[idx[0]] = np.inf
        return out
    return penalty_factor * np.array([_penalty_point(x, recent_points) for x in X])


def _penalise(acq, X, penalty, recent_points, grid_indices, penalty_factor):
    if penalty:
        X_ = grid_indices if grid_indices is not None else X
        acq = acq - compute_penalty(X_, recent_points, penalty, penalty_factor)
    return acq


def _check_penalty(penalty, recent_points):
    if penalty and not isinstance(recent_points, np.ndarray):
        raise ValueError("Please provide an array of recently visited points")


# ------------------------------------------------------------------ model-level functions (acquisition.py)
def _is_bnn(model):
    from .bnn import BNN
    return isinstance(model, BNN)


def _check_bnn(model):
    """the acquisition functions take a fitted one-output BNN"""
    if model.output_dim != 1:
        raise ValueError(f"acquisition functions need a one-output BNN; this one has output_dim={model.output_dim}")
    if model.mcmc is None:
        raise ValueError("the BNN has no posterior samples: fit it first")


def _num_draws(samples):
    """the number of posterior draws: the leading length of the samples' first site"""
    return len(next(iter(samples.values())))


def _acq_for_model(kind, rng_key, model, X, n, noiseless, best_f, param, maximize, **kwargs):
    """acquisition.py:23-36 (_compute_mean_and_var) + the base function.  Fully Bayesian model: the moments are taken
    over the S*n posterior samples (column reduction on the device); viGP-style model: over (mean, var) directly.  BNN:
    over the S values y_sampled[:, p, 0], each of which BNN.predict has already averaged over its n noise draws."""
    if _is_bnn(model):
        _check_bnn(model)
        _, y_sampled = model.predict(rng_key, X, n=n, noiseless=noiseless, **kwargs)
        acq, _, _ = model.ctx.acq_samples(kind, np.asarray(y_sampled)[:, :, 0], best_f, param, maximize)
        return acq
    if getattr(model, "mcmc", None) is not None:
        _, y_sampled = model.predict(rng_key, X, n=n, noiseless=noiseless, **kwargs)
        y = np.asarray(y_sampled, dtype=np.float64).reshape(n * y_sampled.shape[0], -1)
        acq, _, _ = model.ctx.acq_samples(kind, y, best_f, param, maximize)
        return acq
    mean, var = model.predict(rng_key, X, noiseless=noiseless, **kwargs)
    return model.ctx.acq_moments(kind, mean, var, best_f, param, maximize)


def EI(rng_key, model, X, best_f: float = None, maximize: bool = False, n: int = 1, noiseless: bool = False,
       penalty: Optional[str] = None, recent_points=None, grid_indices=None, penalty_factor: float = 1.0, **kwargs):
    """Expected improvement -- gpax/acquisition/acquisition.py:50-143."""
    _check_penalty(penalty, recent_points)
    X = np.asarray(X)
    X = X[:, None] if X.ndim < 2 else X
    acq = _acq_for_model("EI", rng_key, model, X, n, noiseless, best_f, 0.0, maximize, **kwargs)
    return _penalise(acq, X, penalty, recent_points, grid_indices, penalty_factor)


def UCB(rng_key, model, X, beta: float = 0.25, maximize: bool = False, n: int = 1, noiseless: bool = False,
        penalty: Optional[str] = None, recent_points=None, grid_indices=None, penalty_factor: float = 1.0, **kwargs):
    """Upper confidence bound -- acquisition.py:146-227."""
    _check_penalty(penalty, recent_points)
    X = np.asarray(X)
    X = X[:, None] if X.ndim < 2 else X
    acq = _acq_for_model("UCB", rng_key, model, X, n, noiseless, None, beta, maximize, **kwargs)
    return _penalise(acq, X, penalty, recent_points, grid_indices, penalty_factor)


def POI(rng_key, model, X, best_f: float = None, xi: float = 0.01, maximize: bool = False, n: int = 1,
        noiseless: bool = False, penalty: Optional[str] = None, recent_points=None, grid_indices=None,
        penalty_factor: float = 1.0, **kwargs):
    """Probability of improvement -- acquisition.py:230-314."""
    _check_penalty(penalty, recent_points)
    X = np.asarray(X)
    X = X[:, None] if X.ndim < 2 else X
    acq = _acq_for_model("POI", rng_key, model, X, n, noiseless, best_f, xi, maximize, **kwargs)
    return _penalise(acq, X, penalty, recent_points, grid_indices, penalty_factor)


def UE(rng_key, model, X, n: int = 1, noiseless: bool = False, penalty: Optional[str] = None, recent_points=None,
       grid_indices=None, penalty_factor: float = 1.0, **kwargs):
    """Uncertainty-based exploration -- acquisition.py:317-392."""
    _check_penalty(penalty, recent_points)
    X = np.asarray(X)
    X = X[:, None] if X.ndim < 2 else X
    acq = _acq_for_model("UE", rng_key, model, X, n, noiseless, None, 0.0, False, **kwargs)
    return _penalise(acq, X, penalty, recent_points, grid_indices, penalty_factor)


def kg(model, X_new, sample, rng_key=None, n: int = 10, maximize: bool = True, noiseless: bool = True, eps=None, **kwargs):
    """Knowledge gradient for one sample of the hyper-parameters -- base_acq.py:158-232.  One posterior call
    (mean, cov and the n simulated observations y_sim = mean + chol(cov) eps, base_acq.py:221-223) and one closed-form
    rank-1 update kernel instead of P*n re-factorisations.  `eps` [n, P] may be injected (tests); otherwise it follows
    the reference's key: normal(rng_key, (n, P))."""
    X_new = np.asarray(model._set_data(X_new), dtype=np.float64)
    P = X_new.shape[0]
    jitter = float(kwargs.get("jitter", 1e-6))
    # models with a noise per task give the rank-1 update's diagonal terms per candidate (viMTDKL._kg_terms)
    terms = model._kg_terms(X_new, sample, noiseless, jitter) if hasattr(model, "_kg_terms") else None
    if eps is None:
        key = rng_key if rng_key is not None else prng.PRNGKey(0)
        eps = posterior_eps(key, 1, n, P, np.float32, per_draw_keys=False)
    out = model._posterior_batched(X_new, sample, False, noiseless, ("mean", "cov"), eps=np.asarray(eps).reshape(1, n, P), **kwargs)
    mean, cov, ysim = out["mean"][0], out["cov"][0], out["y_sampled"][0]
    if terms is not None:
        return model.ctx.kg(mean, cov, ysim, terms[0], terms[1], maximize)
    kp = sample[1] if isinstance(sample, tuple) else sample          # viDKL's samples: (nn_params, kernel_params)
    noise = float(np.asarray(kp["noise"]))
    diag_sub = noise * (0.0 if noiseless else 1.0) + jitter
    return model.ctx.kg(mean, cov, ysim, diag_sub, noise + jitter, maximize)


def _refuse_kg_on_bnn(model):
    if _is_bnn(model):
        raise ValueError("KG / qKG condition a GP posterior on simulated observations; a BNN would need a refit")


def KG(rng_key, model, X, n: int = 1, maximize: bool = False, noiseless: bool = False, penalty: Optional[str] = None,
       recent_points=None, grid_indices=None, penalty_factor: float = 1.0, **kwargs):
    """Knowledge gradient -- acquisition.py:395-484: kg() for the variational model's parameters, or one row per
    posterior draw ([S, P], the reference's vmap over the draws) for an MCMC model.  Not for a BNN (ValueError): kg()
    conditions a GP posterior on simulated observations, which for a network would mean a refit."""
    _refuse_kg_on_bnn(model)
    _check_penalty(penalty, recent_points)
    X = np.asarray(X)
    X = X[:, None] if X.ndim < 2 else X
    samples = model.get_samples()
    if getattr(model, "mcmc", None) is not None:
        S = len(next(iter(samples.values())))
        keys = prng.split(prng.as_key(rng_key), S)
        vals = []
        for s in range(S):
            one = {k: np.asarray(v)[s] for k, v in samples.items()}
            vals.append(kg(model, X, one, keys[s], n, maximize, noiseless, **kwargs))
        acq = np.stack(vals)
    else:
        acq = kg(model, X, samples, rng_key, n, maximize, noiseless, **kwargs)
    return _penalise(acq, X, penalty, recent_points, grid_indices, penalty_factor)


# ------------------------------------------------------------------ q-batch functions (batch_acquisition.py)
def _subsample(samples, num, rng_key):
    """gpax/utils/utils.py:84-102 (random_sample_dict): `num` consistent rows of every site."""
    N = len(next(iter(samples.values())))
    rng = np.random.default_rng(int(np.asarray(prng.as_key(rng_key), dtype=np.uint64).sum()))
    idx = rng.permutation(N)[:num]
    return {k: np.asarray(v)[idx] for k, v in samples.items()}


def _q_acq(kind, rng_key, model, X, best_f, param, maximize, noiseless, maximize_distance, subsample_size, n_evals,
           indices, **kwargs):
    """batch_acquisition.py:20-57: the acquisition function of `subsample_size` individual posterior draws, one row each
    ([subsample_size, P]); one batched posterior call (mean + diag variance) and one epilogue launch per evaluation.
    BNN: draw s's moments are (loc_s, sigma_s^2), loc from one b2gp_bnn_predict call; noiseless is refused, since one
    weight draw has no spread without its noise."""
    bnn = _is_bnn(model)
    if bnn:
        _check_bnn(model)
        if noiseless:
            raise ValueError("q-batch acquisitions on a BNN need noiseless=False: one weight draw has no spread without noise")
    if getattr(model, "mcmc", None) is None:
        raise ValueError("The model needs to be fully Bayesian")
    X = np.asarray(X)
    X = X[:, None] if X.ndim < 2 else X

    def rows(samples, Xq):
        if bnn:
            loc, _ = model._predict_draws(model._set_data(Xq), np.atleast_2d(model.to_flat(samples)))
            var = np.broadcast_to(np.asarray(samples["noise"], np.float64).reshape(-1, 1) ** 2, loc.shape[:2])
            return model.ctx.acq_moments(kind, loc[:, :, 0], var, best_f, param, maximize)
        out = model._posterior_batched(Xq, samples, True, noiseless, ("mean", "var"), **kwargs)
        return model.ctx.acq_moments(kind, out["mean"], out["var"], best_f, param, maximize)

    return _q_select(rows, rng_key, model, X, maximize_distance, subsample_size, n_evals, indices)


def _q_select(rows, rng_key, model, X, maximize_distance, subsample_size, n_evals, indices):
    """batch_acquisition.py:34-57: rows(samples, X) of one random subsample of the draws, or of the subsample (out of
    n_evals) whose per-draw maximisers lie farthest apart"""
    if not maximize_distance:
        return rows(_subsample(model.get_samples(), subsample_size, rng_key), X)
    X_ = np.asarray(indices) if indices is not None else X
    best, best_d = None, -np.inf
    for sub in prng.split(prng.as_key(rng_key), n_evals):
        acq = rows(_subsample(model.get_samples(), subsample_size, sub), X_)
        d = np.linalg.norm(acq.argmax(-1)).mean()
        if d > best_d:
            best, best_d = acq, d
    return best


def qEI(rng_key, model, X, best_f: float = None, maximize: bool = False, noiseless: bool = False,
        maximize_distance: bool = False, subsample_size: int = 1, n_evals: int = 10, indices=None, **kwargs):
    """batch_acquisition.py:60-118."""
    return _q_acq("EI", rng_key, model, X, best_f, 0.0, maximize, noiseless, maximize_distance, subsample_size, n_evals,
                  indices, **kwargs)


def qUCB(rng_key, model, X, beta: float = 0.25, maximize: bool = False, noiseless: bool = False,
         maximize_distance: bool = False, subsample_size: int = 1, n_evals: int = 10, indices=None, **kwargs):
    """batch_acquisition.py:121-175."""
    return _q_acq("UCB", rng_key, model, X, None, beta, maximize, noiseless, maximize_distance, subsample_size, n_evals,
                  indices, **kwargs)


def qPOI(rng_key, model, X, best_f: float = None, xi: float = 0.01, maximize: bool = False, noiseless: bool = False,
         maximize_distance: bool = False, subsample_size: int = 1, n_evals: int = 10, indices=None, **kwargs):
    """batch_acquisition.py:178-232."""
    return _q_acq("POI", rng_key, model, X, best_f, xi, maximize, noiseless, maximize_distance, subsample_size, n_evals,
                  indices, **kwargs)


def qKG(rng_key, model, X, n: int = 10, maximize: bool = False, noiseless: bool = False, maximize_distance: bool = False,
        subsample_size: int = 1, n_evals: int = 10, indices=None, **kwargs):
    """batch_acquisition.py:235-282: kg() of each sub-sampled posterior draw, one row per draw ([subsample_size, P]),
    with the draw sub-sampling and the `maximize_distance` selection of the other q-batch functions.  Every draw's kg()
    uses `rng_key` for its simulated observations, as the reference's single_acq does.  Not for a BNN (ValueError)."""
    _refuse_kg_on_bnn(model)
    if getattr(model, "mcmc", None) is None:
        raise ValueError("The model needs to be fully Bayesian")
    X = np.asarray(X)
    X = X[:, None] if X.ndim < 2 else X

    def rows(samples, Xq):
        S = len(next(iter(samples.values())))
        return np.stack([kg(model, Xq, {k: np.asarray(v)[s] for k, v in samples.items()}, rng_key, n, maximize, noiseless,
                            **kwargs) for s in range(S)])

    return _q_select(rows, rng_key, model, X, maximize_distance, subsample_size, n_evals, indices)


# ------------------------------------------------------------------ Thompson sampling (acquisition.py:487-524)
def Thompson(rng_key, model, X, n: int = 1, noiseless: bool = False, **kwargs):
    """Thompson sampling -- acquisition.py:487-524.  MCMC model: one hyper-parameter draw picked by
    `prng.randint(rng_key, (1,), 0, S)` (jax.random.randint), then `predict` with that draw and `rng_key`; the n samples
    are averaged when n > 1.  Otherwise the reference calls `model.sample_from_posterior`, which ExactGP and viGP do
    not have (there as here), so they raise AttributeError.  The draws are counted along the samples' first site, so a BNN
    (which has no k_length) works too; its y_sampled [1, P, 1] is already averaged over the n noise draws and comes back
    in the GP's layout, [1, 1, P] for n = 1 and [P] for n > 1."""
    bnn = _is_bnn(model)
    if bnn:
        _check_bnn(model)
    if getattr(model, "mcmc", None) is not None:
        posterior_samples = model.get_samples()
        idx = prng.randint(prng.as_key(rng_key), (1,), 0, _num_draws(posterior_samples))
        samples = {k: np.asarray(v)[idx] for k, v in posterior_samples.items()}
        _, tsample = model.predict(rng_key, X, samples, n, noiseless=noiseless, **kwargs)
        if bnn:
            tsample = np.asarray(tsample)[:, None, :, 0]
        if n > 1:
            tsample = tsample.mean(1).squeeze()
        return tsample
    _, tsample = model.sample_from_posterior(rng_key, X, n=1, noiseless=noiseless, **kwargs)
    return tsample


# ------------------------------------------------------------------ optimize_acq (optimize.py)
def ensure_array(x):
    """optimize.py:91-97: a float becomes [x]; a list, tuple or array becomes an array; anything else (an int included)
    is a TypeError."""
    if isinstance(x, np.ndarray):
        return x
    if isinstance(x, (list, tuple, float)):
        return np.array([x]) if isinstance(x, float) else np.array(x)
    raise TypeError(f"Expected input to be a list, tuple, float, or jnp.ndarray, got {type(x)} instead.")


def _pdf(u):
    return np.exp(-0.5 * u * u - 0.9189385332046727)


def acq_value_grad(kind, mean, var, dmean, dvar, eps=None, best_f=None, param=0.0, maximize=False):
    """Value and gradient w.r.t. x of the acquisition function `kind` ('EI', 'UCB', 'POI', 'UE') at ONE test point x.

    mean, var [S] and dmean, dvar [S, d] are the per-draw posterior moments at x and their gradients.  eps None: S == 1
    and the moments are used directly (the viGP / MAP branch of acquisition.py:35).  eps [S, n]: the reference's
    reparameterised samples y[s, i] = mean[s] + sqrt(var[s]) eps[s, i] (chol of the 1 x 1 covariance is sqrt(var)) are
    pooled into their mean and population variance (acquisition.py:31-34), and both are differentiated through the
    samples.  best_f None is the moments' own mean, as base_acq.py:59-60 takes it over one point, and is differentiated
    too (so EI's u is 0 and its value sigma * phi(0), as jax.grad of the reference gives).  param is beta (UCB) or
    xi (POI).  Returns (value, gradient [d])."""
    from scipy.special import ndtr
    mean, var = np.asarray(mean, np.float64).reshape(-1), np.asarray(var, np.float64).reshape(-1)
    dmean, dvar = np.asarray(dmean, np.float64).reshape(mean.size, -1), np.asarray(dvar, np.float64).reshape(mean.size, -1)
    if eps is None:
        M, V, dM, dV = mean[0], var[0], dmean[0], dvar[0]
    else:
        eps = np.asarray(eps, np.float64).reshape(mean.size, -1)
        sd = np.sqrt(var)
        y = mean[:, None] + sd[:, None] * eps                                        # [S, n]
        dy = dmean[:, None, :] + (dvar / (2.0 * sd[:, None]))[:, None, :] * eps[:, :, None]   # [S, n, d]
        R = y.size
        M = y.mean()
        V = ((y - M) ** 2).mean()
        dM = dy.reshape(R, -1).mean(0)
        dV = 2.0 * ((y - M).reshape(R, 1) * (dy.reshape(R, -1) - dM)).mean(0)
    sigma = np.sqrt(V)
    dsigma = dV / (2.0 * sigma)
    sgn = 1.0 if maximize else -1.0
    if kind == "UE":                                                                 # base_acq.py:129-130
        return sigma, dsigma
    if kind == "UCB":                                                                # base_acq.py:97-103
        delta = np.sqrt(param * V)
        ddelta = param * dV / (2.0 * delta)
        return sgn * M + delta, sgn * dM + ddelta
    best, dbest = (M, dM) if best_f is None else (float(best_f), 0.0)
    if kind == "EI":                                                                 # base_acq.py:59-69
        u = sgn * (M - best) / sigma
        return sigma * (_pdf(u) + u * ndtr(u)), dsigma * _pdf(u) + sgn * ndtr(u) * (dM - dbest)
    if kind == "POI":                                                                # base_acq.py:148-155
        u = sgn * (M - best - param) / sigma
        du = sgn * (dM - dbest) / sigma - u * dsigma / sigma
        return ndtr(u), _pdf(u) * du
    raise ValueError(f"no analytic gradient for {kind}")


# the acquisition functions with an analytic gradient, and the keyword that carries their parameter
_ANALYTIC = {"EI": None, "UCB": "beta", "POI": "xi", "UE": None}
_DEFAULT_PARAM = {"EI": 0.0, "UCB": 0.25, "POI": 0.01, "UE": 0.0}


def _analytic_kind(acq_fn, model, kwargs):
    """'EI' / 'UCB' / 'POI' / 'UE' when acq_fn is one of them and the gradient can be had in closed form, else None.

    A plain ExactGP or viGP qualifies: their predict() is the exact-GP posterior that b2gp_posterior_grad
    differentiates.  So do a plain viDKL or DKL with single-channel targets: their predict() is that posterior on the
    network's embedding, which b2gp_dkl_posterior_grad differentiates w.r.t. the raw inputs.  So does a one-output BNN:
    its samples are loc + sigma * (mean noise draw) per weight draw, and b2gp_bnn_predict_grad differentiates loc.  So
    does a MultiTaskGP in the multitask form (task id in the last column) or a CoregGP, without a mean function: their
    predict() at one point is the LCM posterior that b2gp_posterior_multitask_grad differentiates.  Every other subclass
    (viSparseGP, MeasuredNoiseGP, VarNoiseGP, vExactGP, UIGP, viMTDKL, iBNN, or a user's own) predicts something else,
    so it takes the finite-difference branch even though it inherits _posterior_grad; so do a multi-channel viDKL and
    a MultiTaskGP in the Kronecker form."""
    from .bnn import BNN
    from .dkl import DKL, viDKL
    from .gp import ExactGP
    from .mtgp import CoregGP, MultiTaskGP
    from .vigp import viGP
    kind = {EI: "EI", UCB: "UCB", POI: "POI", UE: "UE"}.get(acq_fn)
    if kind is not None and not kwargs.get("penalty") and type(model) is BNN:
        return kind if model.output_dim == 1 else None
    if kind is not None and not kwargs.get("penalty") and type(model) in (MultiTaskGP, CoregGP):
        return kind if not model.shared_input and model.mean_fn is None else None
    if kind is None or kwargs.get("penalty") or type(model) not in (ExactGP, viGP, viDKL, DKL):
        return None
    if model.mean_fn is not None or model._fused is None:
        return None
    if type(model) in (viDKL, DKL) and getattr(model, "y_train", None) is not None and np.ndim(model.y_train) != 1:
        return None
    return kind


def _analytic_args(kind, kwargs):
    """(the keywords left for the model, n, noiseless, maximize, best_f, param) of acquisition `kind` called with kwargs"""
    kw = dict(kwargs)
    n = int(kw.pop("n", 1))
    noiseless = bool(kw.pop("noiseless", False))
    maximize = bool(kw.pop("maximize", False))
    best_f = kw.pop("best_f", None) if kind in ("EI", "POI") else None
    pname = _ANALYTIC[kind]
    param = float(kw.pop(pname, _DEFAULT_PARAM[kind])) if pname else 0.0
    for k in ("penalty", "recent_points", "grid_indices", "penalty_factor"):
        kw.pop(k, None)
    if kind == "UE":
        maximize = False
    return kw, n, noiseless, maximize, best_f, param


def _analytic_objective(kind, rng_key, model, d, kwargs):
    """x [d] -> (acq(x), d acq / dx) through one model._posterior_grad call per evaluation (b2gp_posterior_grad,
    b2gp_dkl_posterior_grad for viDKL / DKL, or b2gp_posterior_multitask_grad for MultiTaskGP / CoregGP)"""
    from .gp import _eps_dtype
    kw, n, noiseless, maximize, best_f, param = _analytic_args(kind, kwargs)
    mcmc = getattr(model, "mcmc", None) is not None
    samples = model.get_samples()
    S = len(next(iter(samples.values()))) if mcmc else 1
    eps = posterior_eps(rng_key, S, n, 1, _eps_dtype())[:, :, 0] if mcmc else None

    def f(x):
        mean, var, dmean, dvar = model._posterior_grad(np.asarray(x, np.float64).reshape(1, d), samples, mcmc, noiseless, **kw)
        return acq_value_grad(kind, mean[:, 0], var[:, 0], dmean[:, 0, :], dvar[:, 0, :], eps, best_f, param, maximize)
    return f


@contextlib.contextmanager
def _bnn_objective(kind, rng_key, model, d, kwargs):
    """x [d] -> (acq(x), d acq / dx) on a one-output BNN, one b2gp_bnn_predict_grad call per evaluation.  The weight
    sets go to the device once for the whole optimisation.  BNN.predict's samples at one point are y_s = loc_s + sigma_s
    e_s, e_s the mean of the n normals of draw s in the stream predict draws at P = 1 (sigma_s = 0 when noiseless), so
    dy_s = dloc_s; their pooled mean and population variance and those moments' gradients go to acq_value_grad."""
    from ._ffi import ACT_TANH
    from .gp import _eps_dtype
    kw, n, noiseless, maximize, best_f, param = _analytic_args(kind, kwargs)
    samples = kw.get("samples") or model.get_samples()
    flat = np.atleast_2d(model.to_flat(samples))
    S = flat.shape[0]
    eps = np.asarray(posterior_eps(rng_key, S, n, 1, _eps_dtype()), np.float64).reshape(S, n)
    sigma = 0.0 if noiseless else np.asarray(samples["noise"], np.float64).reshape(S)
    e = sigma * (eps.sum(1) / n)
    ctx = model.ctx
    Pd, Xd = ctx.to_device(flat), ctx.alloc((1, d))
    try:
        def f(x):
            Xd.upload(np.asarray(x, np.float64).reshape(1, d))
            loc, dloc = ctx.bnn_predict_grad(Xd, model.widths, ACT_TANH, Pd)
            y, dy = loc[:, 0] + e, dloc[:, 0, :]
            M = y.mean()
            dM = dy.mean(0)
            V = ((y - M) ** 2).mean()
            dV = 2.0 * ((y - M)[:, None] * (dy - dM)).mean(0)
            return acq_value_grad(kind, [M], [V], dM[None], dV[None], None, best_f, param, maximize)
        yield f
    finally:
        Pd.free()
        Xd.free()


def optimize_acq(rng_key, model, acq_fn, num_initial_guesses: int, lower_bound, upper_bound, **kwargs):
    """Maximise `acq_fn` over the box [lower_bound, upper_bound] -- gpax/acquisition/optimize.py:19-88.

    The acquisition is evaluated at `num_initial_guesses` uniform points (jax.random.uniform on `rng_key`, float32
    unless x64 is enabled), and L-BFGS-B (scipy.optimize.minimize, the routine jaxopt's ScipyBoundedMinimize wraps;
    maxiter 500 as jaxopt's default) minimises -acq(x) from the best of them, x shaped (1, d) for each evaluation.

    The reference differentiates the acquisition w.r.t. x with JAX.  Here EI, UCB, POI and UE without a penalty, on a
    plain ExactGP / viGP with a built-in kernel and no mean function, get the same gradient in closed form from the
    posterior's own derivatives w.r.t. the test input (b2gp_posterior_grad: one posterior call per evaluation, value and
    gradient together).  On a viDKL or DKL with single-channel targets the posterior's gradient w.r.t. the embedding is
    pulled back through the network to the raw input (b2gp_dkl_posterior_grad, one call per evaluation); viDKL's single
    weight set keeps the factor of the training embedding cached across the evaluations.  On a one-output BNN the
    network's gradient w.r.t. the input comes from b2gp_bnn_predict_grad, one call per evaluation with the weight sets
    resident on the device for the whole run.  On a MultiTaskGP in the multitask form or a CoregGP the LCM posterior's
    gradient comes from b2gp_posterior_multitask_grad, one call per evaluation, with 0 on the task column (the
    reference's astype(int) passes no gradient; fix the task by equal lower and upper bounds).  Every other acquisition
    (KG, Thompson, the q-batch functions, penalties, user callables), model (mean functions, viMTDKL, multi-channel
    viDKL, the Kronecker form of MultiTaskGP, iBNN, other subclasses) is handed to L-BFGS-B without a gradient: SciPy
    then takes finite differences, d + 1 posterior calls per gradient.  Returns the maximiser with the shape of the reference's `result.params`: that of the squeezed best initial
    guess, [d], or a 0-d array in one dimension."""
    from scipy.optimize import minimize
    from .utils import x64_enabled
    lower_bound = ensure_array(lower_bound)
    upper_bound = ensure_array(upper_bound)
    dt = np.float64 if x64_enabled() else np.float32
    d = lower_bound.shape[0]
    guesses = prng.uniform(prng.as_key(rng_key), (num_initial_guesses, d), dt,
                           np.asarray(lower_bound, dt), np.asarray(upper_bound, dt))
    initial_acq_vals = np.asarray(acq_fn(rng_key, model, guesses, **kwargs))
    x0 = np.asarray(guesses[initial_acq_vals.argmax()]).squeeze()
    shape = x0.shape
    bounds = list(zip(np.broadcast_to(lower_bound, (d,)).astype(float), np.broadcast_to(upper_bound, (d,)).astype(float)))
    kind = _analytic_kind(acq_fn, model, kwargs)
    if kind is not None:
        objective = (_bnn_objective(kind, rng_key, model, d, kwargs) if _is_bnn(model)
                     else contextlib.nullcontext(_analytic_objective(kind, rng_key, model, d, kwargs)))
        with objective as f:
            def fun(x):
                v, g = f(x)
                return -float(v), -np.asarray(g, np.float64).reshape(-1)
            res = minimize(fun, np.asarray(x0, np.float64).reshape(-1), jac=True, method="L-BFGS-B", bounds=bounds,
                           options={"maxiter": 500})
    else:
        def fun(x):   # optimize.py:70-74
            x = np.array([x]).reshape(1, -1)
            return -float(np.asarray(acq_fn(rng_key, model, x, **kwargs)).reshape(()))
        res = minimize(fun, np.asarray(x0, np.float64).reshape(-1), jac=None, method="L-BFGS-B", bounds=bounds,
                       options={"maxiter": 500})
    return np.asarray(res.x, dtype=dt).reshape(shape)
