"""
diagnostics.py -- the convergence diagnostics hypothesis learning restarts on (numpyro.diagnostics.gelman_rubin /
split_gelman_rubin, which gpax/hypo.py:75-93 calls), on NumPy arrays.
"""
import numpy as np


def gelman_rubin(x) -> np.ndarray:
    """R-hat of draws x [chains, draws, ...] (at least 2 chains of 2 draws): sqrt(((n - 1) / n W + B / n) / W), with W
    the mean over chains of the within-chain variances and B / n the variance of the chain means (both ddof 1).
    Returns one value per trailing element (a 0-d array for a scalar site)."""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim < 2 or x.shape[0] < 2 or x.shape[1] < 2:
        raise ValueError(f"gelman_rubin needs [chains >= 2, draws >= 2, ...]; got shape {x.shape}")
    n = x.shape[1]
    w = x.var(axis=1, ddof=1).mean(axis=0)
    b_n = x.mean(axis=1).var(axis=0, ddof=1)
    return np.sqrt(((n - 1) / n * w + b_n) / w)


def split_gelman_rubin(x) -> np.ndarray:
    """R-hat with every chain split in halves: the first n // 2 and the last n // 2 draws of each of the C chains of
    x [C, n, ...] become 2C chains (n >= 4), so that one chain that drifts is caught too"""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim < 2 or x.shape[1] < 4:
        raise ValueError(f"split_gelman_rubin needs [chains, draws >= 4, ...]; got shape {x.shape}")
    half = x.shape[1] // 2
    return gelman_rubin(np.concatenate([x[:, :half], x[:, -half:]], axis=0))
