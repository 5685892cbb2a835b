"""bnn_time.py -- time BNN's two GPU entry points on both routes and one BNN.fit, and print one JSON line.

  loglik    per-evaluation wall time of b2gp_bnn_loglik (value + all gradients; the call returns after its device work)
            with X and y device-resident, [64, 32] network, D in {1, 16}, O = 1, N in {64, 512, 4096, 65536}; fused and
            layered alternate call by call (`--reps` rounds of `--inner` calls each), median and minimum per call
  predict   b2gp_bnn_predict with S = 2000 draws, n = 1, P in {1000, 10000}, D = 1, both routes alternating
  kernels   in a run of its own, torch.profiler's device time per call of bnn_loglik_tile_kernel and bnn_reduce_kernel
            (fused route, default network, D = 1, O = 1, N in {512, 4096, 65536}, 20 calls)
  fit       wall time and likelihood-evaluation count of one BNN.fit (default network, N = 256, 200 + 200 draws)
Records the card's name, power limit and SM clock in the same process."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpax_b200  # noqa: E402
from tools.dkl_time import card, kernel_times  # noqa: E402

TANH = 1


def alternate(ctx, fns, reps):
    """{route: {median_ms, min_ms}} over `reps` rounds, the routes alternating inside each round"""
    ts = {k: [] for k in fns}
    for k, f in fns.items():          # warm-up: module load, allocations
        with ctx.options(bnn_fused=k == "fused"):
            f()
    for _ in range(reps):
        for k, f in fns.items():
            with ctx.options(bnn_fused=k == "fused"):
                t0 = time.perf_counter()
                n = f()
                ts[k].append((time.perf_counter() - t0) * 1e3 / n)
    return {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v))} for k, v in ts.items()}


def loglik_kernel_times(ctx, rows=(512, 4096, 65536), calls=20):
    """[{N, tile_ms, reduce_ms}]: device time per call of the fused route's two kernels at the default shape"""
    rng = np.random.default_rng(1)
    widths = [64, 32, 1]
    npar = sum(i * w + w for i, w in zip([1] + widths[:-1], widths))
    out = []
    for N in rows:
        X = rng.uniform(-1, 1, (N, 1))
        y = np.sin(3 * X) + 0.1 * rng.standard_normal((N, 1))
        flat = 0.3 * rng.standard_normal(npar)
        Xd, yd = ctx.to_device(X), ctx.to_device(y)
        ctx.bnn_loglik(Xd, yd, widths, TANH, flat, 0.2)

        def run():
            for _ in range(calls):
                ctx.bnn_loglik(Xd, yd, widths, TANH, flat, 0.2)
        t = kernel_times(run)
        out.append({"N": N, "tile_ms": t.get("bnn_loglik_tile_kernel", 0.0) / calls,
                    "reduce_ms": t.get("bnn_reduce_kernel", 0.0) / calls})
        Xd.free()
        yd.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--inner", type=int, default=20)
    ap.add_argument("--rows", default="64,512,4096,65536")
    ap.add_argument("--fit-draws", type=int, default=200)
    ap.add_argument("--kernels-only", action="store_true", help="only the profiled kernel times")
    a = ap.parse_args()
    ctx = gpax_b200.default_context()
    if a.kernels_only:
        print(json.dumps({"card": card(), "kernels": loglik_kernel_times(ctx)}))
        return
    rng = np.random.default_rng(0)
    res = {"card": card(), "loglik": [], "predict": []}
    hidden = [64, 32]
    for D in (1, 16):
        for N in [int(v) for v in a.rows.split(",")]:
            widths = hidden + [1]
            npar = sum(i * w + w for i, w in zip([D] + widths[:-1], widths))
            X = rng.uniform(-1, 1, (N, D))
            y = np.sin(3 * X[:, :1]) + 0.1 * rng.standard_normal((N, 1))
            flat = 0.3 * rng.standard_normal(npar)
            Xd, yd = ctx.to_device(X), ctx.to_device(y)

            def run(Xd=Xd, yd=yd, widths=widths, flat=flat):
                for _ in range(a.inner):
                    ctx.bnn_loglik(Xd, yd, widths, TANH, flat, 0.2)
                return a.inner
            t = alternate(ctx, {"fused": run, "layered": run}, a.reps)
            res["loglik"].append({"D": D, "N": N, "O": 1, **{f"{k}_{m}": v[m] for k, v in t.items() for m in v}})
            Xd.free()
            yd.free()
    widths = hidden + [1]
    npar = sum(i * w + w for i, w in zip([1] + widths[:-1], widths))
    S = 2000
    flats = 0.5 * rng.standard_normal((S, npar))
    sig = rng.uniform(0.05, 0.3, S)
    for Pn in (1000, 10000):
        X = rng.uniform(-1, 1, (Pn, 1))
        eps = rng.standard_normal((S, 1, Pn, 1))

        def run_p(X=X, eps=eps):
            ctx.bnn_predict(X, widths, TANH, flats, sig, eps)
            return 1
        t = alternate(ctx, {"fused": run_p, "layered": run_p}, max(2, a.reps // 2))
        res["predict"].append({"S": S, "P": Pn, **{f"{k}_{m}": v[m] for k, v in t.items() for m in v}})
    X = np.sort(rng.uniform(-2, 2, 256))
    y = np.sin(2 * X) + 0.1 * rng.standard_normal(256)
    m = gpax_b200.BNN(1, 1, ctx=ctx)
    t0 = time.perf_counter()
    m.fit(0, X, y, num_warmup=a.fit_draws, num_samples=a.fit_draws, progress_bar=False, print_summary=False)
    wall = time.perf_counter() - t0
    ev = m.mcmc.stats[0]["grad_evals"]
    res["fit"] = {"N": 256, "warmup": a.fit_draws, "samples": a.fit_draws, "wall_s": wall, "grad_evals": ev,
                  "ms_per_eval": 1e3 * wall / ev}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
