"""
hypo.py -- hypothesis learning (arXiv:2112.06649) with the reference's surface (gpax/hypo.py:21-167): fit one candidate
physical model to the measurements with `step`, keep the one whose predictions are most uncertain, and choose the next
model by a bandit policy (`sample_next`, `softmax`, `eps_greedy`) over the running rewards kept by `update_record`.

`step(gp_wrap=True)` fits an ExactGP with the candidate as its mean function on the GPU likelihood (b2gp_mll) and
predicts on the GPU posterior; `step(gp_wrap=False)` fits the standalone sPM on the host.

One deliberate divergence: the restart test takes the maximum split r-hat over every component of every site.  The
reference calls `.item()` on each site's r-hat and so raises on a vector site such as a multi-dimensional `k_length`
(gp_wrap=True with gp_input_dim > 1); for scalar sites the two agree.

The bandit policies draw from NumPy's global generator, as the reference's do: seed it with np.random.seed.
"""
from typing import Callable, Optional

import numpy as np

from .diagnostics import split_gelman_rubin
from .gp import ExactGP
from .spm import sPM
from .utils import get_keys

RHAT_MAX = 1.1


def step(model: Callable, model_prior: Callable, X_measured, y_measured, X_unmeasured=None,
         gp_wrap: Optional[bool] = False, noise_prior: Optional[Callable] = None, gp_kernel: str = "Matern",
         gp_kernel_prior: Optional[Callable] = None, gp_input_dim: Optional[int] = 1,
         num_warmup: Optional[int] = 2000, num_samples: Optional[int] = 2000, num_chains: Optional[int] = 1,
         num_restarts: Optional[int] = 1, print_summary: Optional[bool] = True):
    """
    Fit one candidate model and measure its predictive uncertainty over the unmeasured points (hypo.py:21-99).

    Fit i (i = 0 .. num_restarts - 1) uses the keys get_keys(i); fitting stops at the first fit whose largest split
    r-hat over the sites (all but `mu`) is below 1.1.  gp_wrap=True wraps the model in
    ExactGP(gp_input_dim, gp_kernel, model, gp_kernel_prior, model_prior, noise_prior), gp_wrap=False uses
    sPM(model, model_prior, noise_prior).

    Returns (obj, fitted model): obj is the variance over posterior draws of the predictive samples at X_unmeasured,
    `predict(rng_key, X_unmeasured)` with the last fit's key, [P]; 0 without X_unmeasured.
    """
    for i in range(num_restarts):
        rng_key, _ = get_keys(i)
        if gp_wrap:
            fitted = ExactGP(gp_input_dim, gp_kernel, model, gp_kernel_prior, model_prior, noise_prior)
        else:
            fitted = sPM(model, model_prior, noise_prior)
        fitted.fit(rng_key, X_measured, y_measured, num_warmup, num_samples, num_chains, print_summary=print_summary)
        rhat = max(float(np.max(split_gelman_rubin(v))) for k, v in fitted.get_samples(1).items() if k != "mu")
        if rhat < RHAT_MAX:
            break
    obj = 0
    if X_unmeasured is not None:
        _, samples = fitted.predict(rng_key, X_unmeasured)
        obj = np.asarray(samples).squeeze().var(0)
    return obj, fitted


def sample_next(rewards, method: Optional[str] = "softmax", temperature: Optional[float] = 1.0,
                eps: Optional[float] = 0.4) -> int:
    """
    The index of the model (or input channel) to try next (hypo.py:102-131): `method` 'softmax' (with `temperature`)
    or 'eps-greedy' (with `eps`) over the running rewards [M].  NotImplementedError for another method,
    AttributeError when rewards is not 1-D.
    """
    if method not in ("softmax", "eps-greedy"):
        raise NotImplementedError(f"unknown selection method {method!r}: use 'softmax' or 'eps-greedy'")
    if rewards.ndim != 1:
        raise AttributeError(f"rewards must be a 1-D array; got {rewards.ndim} dimensions")
    if method == "softmax":
        return softmax(rewards, temperature)
    return eps_greedy(rewards, eps)


def softmax(logits, temperature: Optional[float] = 1.0) -> int:
    """Softmax selection (hypo.py:134-143; Zai & Brown, Deep reinforcement learning in action, 2020): index m with
    probability exp(logits_m / T) / sum exp(logits / T), drawn by np.random.choice"""
    w = np.exp(np.asarray(logits) / temperature)
    return np.random.choice(np.arange(len(logits)), p=w / np.sum(w))


def eps_greedy(rewards, eps: Optional[float] = 0.4) -> int:
    """Epsilon-greedy selection (hypo.py:146-156): the best reward's index when np.random.random() > eps, otherwise an
    index uniform over the models (np.random.randint)"""
    if np.random.random() > eps:
        return rewards.argmax()
    return np.random.randint(len(rewards))


def update_record(record: np.ndarray, action: int, r) -> np.ndarray:
    """The running record (hypo.py:159-167): record[m] = (times model m was chosen, its mean reward); choosing
    `action` with reward r updates that row's count and mean in place and returns the record"""
    count, mean = record[action, 0], record[action, 1]
    record[action, 1] = (count * mean + r) / (count + 1)
    record[action, 0] += 1
    return record
