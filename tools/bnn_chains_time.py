"""bnn_chains_time.py -- b2gp_bnn_loglik_draws against S b2gp_bnn_loglik calls, and BNN fits under chain_method
"sequential" against "vectorized" (DESIGN.md 4.19).

  python tools/bnn_chains_time.py [--reps R] [--fit-iters K] [--fit-reps F]

Prints the card, its power limit and its max SM clock first, then one line per measurement.  Likelihood times are host
clocks around calls that end in a device synchronise (every call returns host outputs), best of R after a warm-up of every
shape, with X and y resident on the device as in a fit; `dev` is the device time of the draws call (b2gp_last_timing).
Fit times alternate the two chain methods, and each pair checks that both gave the same samples bit for bit; `lib` is the
host time spent inside the likelihood calls, the rest is the host NUTS loop."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TANH = 1


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
    from gpax_b200 import BNN
    rng = np.random.default_rng(0)
    m = BNN(1, 1)                                       # the default [64, 32] network
    P = m._weight_mask().size
    for N in (64, 256, 4096, 65536):
        X = rng.uniform(-2, 2, (N, 1))
        y = np.sin(1.5 * X) + 0.05 * rng.standard_normal((N, 1))
        Xd, yd = ctx.to_device(X), ctx.to_device(y)
        for S in (1, 4, 8, 16):
            params = 0.3 * rng.standard_normal((S, P))
            sigma = rng.uniform(0.05, 0.5, S)
            loop = best(lambda: [ctx.bnn_loglik(Xd, yd, m.widths, TANH, params[s], sigma[s]) for s in range(S)], reps)
            one = best(lambda: ctx.bnn_loglik_draws(Xd, yd, m.widths, TANH, params, sigma), reps)
            dev = ctx.last_timing()["total_ms"]
            print(f"bnn_loglik_draws N={N:6d} S={S:2d}: {S:2d} x bnn_loglik {loop * 1e3:8.3f} ms   draws {one * 1e3:8.3f} ms "
                  f"(dev {dev:7.3f} ms)   {loop / one:5.2f}x", flush=True)
        Xd.free()
        yd.free()


def fits(ctx, iters, reps):
    import gpax_b200
    rng = np.random.default_rng(4)
    N, chains = 256, 4
    X = np.sort(rng.uniform(-2, 2, N))
    y = np.sin(1.5 * X) + 0.05 * rng.standard_normal(N)
    t = {"sequential": [], "vectorized": []}
    lib = {"sequential": [], "vectorized": []}
    rounds = {}
    for rep in range(reps):
        got = {}
        for method in ("sequential", "vectorized") if rep % 2 == 0 else ("vectorized", "sequential"):
            m = gpax_b200.BNN(1, 1, ctx=ctx)
            spent, calls = [0.0], [0]
            name = "bnn_loglik_draws" if method == "vectorized" else "bnn_loglik"

            def timed(*a, _f=getattr(ctx, name), **kw):
                t0 = time.perf_counter()
                out = _f(*a, **kw)
                spent[0] += time.perf_counter() - t0
                calls[0] += 1
                return out
            setattr(ctx, name, timed)
            try:
                t0 = time.perf_counter()
                m.fit(0, X, y, num_warmup=iters, num_samples=iters, num_chains=chains, chain_method=method,
                      progress_bar=False, print_summary=False)
                t[method].append(time.perf_counter() - t0)
            finally:
                delattr(ctx, name)
            lib[method].append(spent[0])
            rounds[method] = calls[0]
            got[method] = m.get_samples(chain_dim=True)
        same = all(np.array_equal(got["sequential"][k], got["vectorized"][k]) for k in got["sequential"])
        print(f"fit BNN N={N} chains={chains} pair {rep}: sequential {t['sequential'][-1]:7.2f} s (lib {lib['sequential'][-1]:6.2f} s)"
              f"   vectorized {t['vectorized'][-1]:7.2f} s (lib {lib['vectorized'][-1]:6.2f} s)   identical={same}", flush=True)
    ts, tv = min(t["sequential"]), min(t["vectorized"])
    print(f"fit BNN N={N} chains={chains} best: sequential {ts:7.2f} s   vectorized {tv:7.2f} s   {ts / tv:5.2f}x   "
          f"{rounds['sequential']} bnn_loglik calls, {rounds['vectorized']} bnn_loglik_draws calls", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--fit-iters", type=int, default=15)
    ap.add_argument("--fit-reps", type=int, default=2)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    from gpax_b200 import _ffi
    ctx = _ffi.Context(0)
    likelihoods(ctx, a.reps)
    fits(ctx, a.fit_iters, a.fit_reps)
    ctx.close()


if __name__ == "__main__":
    main()
