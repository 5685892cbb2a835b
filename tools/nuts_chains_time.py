"""Times lock-step likelihood draws and vectorized NUTS chains (DESIGN.md 4.15).

  draws  one ctx.mll_draws call over S draws against S ctx.mll calls, wall time per call (median of alternated
         repetitions) and kernel launches per call, N in {32, 96, 256, 1024, 4096}, S in {1, 2, 4, 8}, RBF and NNGP-erf
  fit    ExactGP.fit wall time (RBF, d = 1, 200 + 200 draws) with num_chains in {1, 4, 8} under chain_method
         "sequential" and "vectorized", N in {64, 512}; the two methods alternate and give the same samples

Both arms run in the same process.  Prints the card and its power limit, then one JSON line per row.
usage: python tools/nuts_chains_time.py [--only draws|fit]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def draws_rows(ctx):
    for kind in ("RBF", "NNGP_erf"):
        for N in (32, 96, 256, 1024, 4096):
            rng = np.random.default_rng(N)
            X = rng.uniform(0, 1, (N, 2))
            y = np.sin(5 * X[:, 0]) + 0.1 * rng.standard_normal(N)
            reps = 30 if N <= 256 else (8 if N <= 1024 else 3)
            for S in (1, 2, 4, 8):
                if kind == "RBF":
                    th = np.column_stack([rng.uniform(0.2, 0.4, (S, 2)), np.ones(S), np.full(S, 0.05), np.ones(S)])
                else:
                    th = np.column_stack([np.full(S, 2.0), np.zeros(S), rng.uniform(0.8, 1.2, S), np.full(S, 0.05), np.full(S, 0.1)])
                t_draws, t_loop = [], []
                for r in range(reps + 1):          # the first round warms both arms up
                    for arm in ((0, 1) if r % 2 == 0 else (1, 0)):
                        t0 = time.perf_counter()
                        if arm == 0:
                            ctx.mll_draws(kind, X, y, th)
                            lw = ctx.last_timing()["launches"]
                        else:
                            lm = 0
                            for s in range(S):
                                ctx.mll(kind, X, y, th[s])
                                lm += ctx.last_timing()["launches"]
                        dt = (time.perf_counter() - t0) * 1e3
                        if r > 0:
                            (t_draws if arm == 0 else t_loop).append(dt)
                a, b = float(np.median(t_draws)), float(np.median(t_loop))
                print(json.dumps({"table": "draws", "kind": kind, "N": N, "S": S, "mll_draws_ms": round(a, 3),
                                  "S_x_mll_ms": round(b, 3), "speedup": round(b / a, 2), "launches_draws": lw,
                                  "launches_S_x_mll": lm}), flush=True)


def fit_rows(ctx):
    import gpax_b200
    for N in (64, 512):
        rng = np.random.default_rng(N)
        X = rng.uniform(0, 1, N)
        y = np.sin(6 * X) + 0.1 * rng.standard_normal(N)
        for chains in (1, 4, 8):
            out, samples = {}, {}
            for method in (("sequential", "vectorized") if chains % 8 else ("vectorized", "sequential")):
                m = gpax_b200.ExactGP(1, "RBF", ctx=ctx)
                t0 = time.perf_counter()
                m.fit(0, X, y, num_warmup=200, num_samples=200, num_chains=chains, chain_method=method, progress_bar=False,
                      print_summary=False)
                out[method] = time.perf_counter() - t0
                samples[method] = m.mcmc.get_samples(group_by_chain=True)["k_length"]
                evals = m.mcmc.stats[-1]["grad_evals"]
            print(json.dumps({"table": "fit", "N": N, "chains": chains, "sequential_s": round(out["sequential"], 2),
                              "vectorized_s": round(out["vectorized"], 2),
                              "speedup": round(out["sequential"] / out["vectorized"], 2), "grad_evals": int(evals),
                              "same_samples": bool(np.array_equal(samples["sequential"], samples["vectorized"]))}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=("draws", "fit"))
    a = ap.parse_args()
    from gpax_b200 import _ffi
    print("card, power limit:", card(), flush=True)
    ctx = _ffi.Context(0)
    if a.only in (None, "draws"):
        draws_rows(ctx)
    if a.only in (None, "fit"):
        fit_rows(ctx)
    ctx.close()


if __name__ == "__main__":
    main()
