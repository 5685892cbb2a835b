"""Times sPM.fit and hypo.step (DESIGN.md section 7, row f5).

  fit   sPM.fit wall time of the power-law model a * x**b (LogNormal / Normal priors, LogNormal noise), 200 + 200 draws,
        N in {32, 256}, num_chains in {1, 4} (sequential), with the log-joint evaluations, the model calls and the
        wall time per evaluation
  step  hypo.step wall time on the same model, N = 32 measured and 200 unmeasured points, 200 + 200 draws, one chain,
        gp_wrap=False (sPM, host) and gp_wrap=True (ExactGP with the model as mean function, likelihood on the GPU)

Prints the card and its power limit, then one JSON line per row.
usage: python tools/spm_time.py [--only fit|step]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from gpax_b200 import priors as numpyro  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def model(x, params):
    return params["a"] * x ** params["b"]


def model_priors():
    a = numpyro.sample("a", numpyro.distributions.LogNormal(0, 1))
    b = numpyro.sample("b", numpyro.distributions.Normal(3, 1))
    return {"a": a, "b": b}


def data(N, seed=0):
    rng = np.random.default_rng(seed)
    X = np.linspace(1, 2, N)
    return X, 10 * X ** 2 + 0.1 * rng.standard_normal(N)


def fit_rows():
    import gpax_b200.spm as spm
    from gpax_b200.utils import get_keys
    for N in (32, 256):
        X, y = data(N)
        for chains in (1, 4):
            m = spm.sPM(model, model_priors)
            calls = [0]

            def counted(x, params):
                calls[0] += 1
                return model(x, params)
            m._model = counted
            t0 = time.perf_counter()
            m.fit(get_keys(0)[0], X, y, num_warmup=200, num_samples=200, num_chains=chains, progress_bar=False,
                  print_summary=False)
            dt = time.perf_counter() - t0
            evals = m.mcmc.stats[-1]["grad_evals"]
            print(json.dumps({"table": "fit", "N": N, "chains": chains, "fit_s": round(dt, 3), "evals": evals,
                              "model_calls": calls[0], "us_per_eval": round(dt / evals * 1e6, 1)}), flush=True)


def step_rows():
    from gpax_b200.hypo import step
    X, y = data(32)
    Xu = np.linspace(1, 3, 200)
    for gp_wrap in (False, True):
        if gp_wrap:                                  # the first GPU call pays for context creation: not timed
            step(model, model_priors, X, y, Xu, gp_wrap=True, num_warmup=5, num_samples=5, print_summary=False)
        t0 = time.perf_counter()
        obj, m = step(model, model_priors, X, y, Xu, gp_wrap=gp_wrap, num_warmup=200, num_samples=200,
                      print_summary=False)
        dt = time.perf_counter() - t0
        print(json.dumps({"table": "step", "gp_wrap": gp_wrap, "N": 32, "P": 200, "step_s": round(dt, 3),
                          "obj_mean": float(np.mean(obj))}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["fit", "step"])
    a = ap.parse_args()
    print(f"# card: {card()}", flush=True)
    if a.only in (None, "fit"):
        fit_rows()
    if a.only in (None, "step"):
        step_rows()


if __name__ == "__main__":
    main()
