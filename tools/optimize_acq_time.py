"""Time one optimize_acq evaluation (value + analytic gradient of EI through b2gp_posterior_grad) for a viGP, with and
without factor-cache hits, and the achieved HBM bandwidth of gram_dx_kernel (8 P d N bytes written over its kernel time
from torch.profiler).  Prints one JSON line; needs a GPU.

    python tools/optimize_acq_time.py [--reps 20] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def eval_times(ctx, N, d, reps):
    from gpax_b200 import acquisition as acq, viGP
    rng = np.random.default_rng(N)
    X = rng.uniform(-2, 2, (N, d))
    y = np.sin(X).sum(1) + 0.05 * rng.standard_normal(N)
    v = viGP(d, "RBF", ctx=ctx)
    v.X_train, v.y_train = X, y
    v.kernel_params = {"k_length": np.full(d, 0.8), "k_scale": 1.0, "noise": 0.01}
    f = acq._analytic_objective("EI", 0, v, d, {})
    xs = rng.uniform(-2, 2, (reps, d))
    out = {}
    for cached in (True, False):
        f(xs[0])                                   # warm-up (and, for the cached case, the factor)
        ts = []
        for x in xs:
            if not cached:
                ctx.set_option("drop_factor_cache", 1)
            t0 = time.perf_counter()
            f(x)                                   # returns host values: the call ends in a device synchronise
            ts.append(time.perf_counter() - t0)
        out["cache_hit" if cached else "no_cache"] = {"median_ms": 1e3 * float(np.median(ts)), "min_ms": 1e3 * float(np.min(ts))}
    return out


def gram_dx_bandwidth(ctx, kernel, N=16384, P=512, d=3):
    import torch
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(0)
    X, Xn = rng.uniform(0, 1, (N, d)), rng.uniform(0, 1, (P, d))
    y = rng.standard_normal(N)
    theta = np.array([[0.3] * d + [1.0, 0.01, 1.0]])
    ctx.posterior_grad(kernel, X, y, Xn, theta)                  # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            ctx.set_option("drop_factor_cache", 1)
            ctx.posterior_grad(kernel, X, y, Xn, theta)
        torch.cuda.synchronize()
    us = [getattr(e, "device_time", None) or e.cuda_time for e in prof.events() if "gram_dx_kernel" in e.name]
    if not us:
        raise RuntimeError("torch.profiler recorded no gram_dx_kernel")
    sec = float(np.median(us)) * 1e-6
    nbytes = 8.0 * P * d * N
    return {"kernel": kernel, "N": N, "P": P, "d": d, "kernel_us": sec * 1e6, "bytes_written": nbytes, "GB_per_s": nbytes / sec / 1e9,
            "launches_seen": len(us)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from gpax_b200 import _ffi
    ctx = _ffi.Context(0)
    res = {"gpu": gpu_info(), "d": 3, "acq": "EI", "model": "viGP RBF"}
    for N in (2048, 16384):
        res[f"eval_N{N}"] = eval_times(ctx, N, 3, a.reps)
    res["gram_dx"] = [gram_dx_bandwidth(ctx, k) for k in ("Matern", "Periodic")]
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
