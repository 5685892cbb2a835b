"""noise_chains_time.py -- b2gp_mll_draws_v against S b2gp_mll_v calls, and MeasuredNoiseGP / VarNoiseGP fits under
chain_method "sequential" against "vectorized" (DESIGN.md 4.18).

  python tools/noise_chains_time.py [--reps R] [--fit-iters K]

Prints the card and its power limit first, then one line per measurement.  Likelihood times are host clocks around
calls that end in a device synchronise (every call returns host outputs), best of R after a warm-up of every shape.
Fit times alternate the two chain methods, and each pair checks that both gave the same samples bit for bit."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("no GPU: " + q.stderr)
    return q.stdout.strip()


def best(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return min(ts)


def likelihoods(ctx, reps):
    rng = np.random.default_rng(0)
    for N in (32, 96, 256, 1024):
        X = rng.uniform(0, 1, (N, 1))
        for S in (1, 4, 8):
            Y = np.sin(6 * X[:, 0])[None] + 0.1 * rng.standard_normal((S, N))
            NV = np.exp(rng.normal(-3, 0.5, (S, N)))
            TH = np.column_stack([rng.uniform(0.2, 0.4, S), np.ones(S), np.zeros(S), np.ones(S)])
            loop = best(lambda: [ctx.mll("RBF", X, Y[s], TH[s], 1e-6, True, False, NV[s]) for s in range(S)], reps)
            one = best(lambda: ctx.mll_draws_v("RBF", X, Y, TH, NV, 1e-6, True), reps)
            print(f"mll_draws_v RBF N={N:5d} S={S}: {S} x mll_v {loop * 1e3:8.3f} ms   draws_v {one * 1e3:8.3f} ms   "
                  f"{loop / one:5.2f}x", flush=True)


def fits(ctx, iters):
    import gpax_b200
    rng = np.random.default_rng(4)
    for N in (32, 128):
        X = np.sort(rng.uniform(0, 1, N))[:, None]
        sd = 0.05 + 0.25 * X[:, 0]
        y = np.sin(6 * X[:, 0]) + sd * rng.standard_normal(N)
        for name in ("MeasuredNoiseGP", "VarNoiseGP"):
            for chains in (1, 4, 8):
                t = {"sequential": [], "vectorized": []}
                got = {}
                for rep in range(2):
                    for method in ("sequential", "vectorized") if rep == 0 else ("vectorized", "sequential"):
                        if name == "MeasuredNoiseGP":
                            m, args = gpax_b200.MeasuredNoiseGP(1, "RBF", ctx=ctx), (X, y, sd ** 2)
                        else:
                            m, args = gpax_b200.VarNoiseGP(1, "RBF", ctx=ctx), (X, y)
                        t0 = time.perf_counter()
                        m.fit(0, *args, num_warmup=iters, num_samples=iters, num_chains=chains, chain_method=method,
                              progress_bar=False, print_summary=False)
                        t[method].append(time.perf_counter() - t0)
                        got[method] = m.mcmc.get_samples(group_by_chain=True)
                same = all(np.array_equal(got["sequential"][k], got["vectorized"][k]) for k in got["sequential"])
                ts, tv = min(t["sequential"]), min(t["vectorized"])
                print(f"fit {name:15s} N={N:4d} chains={chains}: sequential {ts:7.2f} s   vectorized {tv:7.2f} s   "
                      f"{ts / tv:5.2f}x   identical={same}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--fit-iters", type=int, default=50)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    from gpax_b200 import _ffi
    ctx = _ffi.Context(0)
    likelihoods(ctx, a.reps)
    fits(ctx, a.fit_iters)
    ctx.close()


if __name__ == "__main__":
    main()
