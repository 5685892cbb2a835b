"""mtgp_time.py -- time the multi-task posterior and likelihood against ExactGP's at the same matrix size; print one JSON line.

  posterior  mean + var of S = 8 draws (b2gp_posterior_multitask / b2gp_posterior)
  mll        value + gradient (b2gp_mll_multitask / b2gp_mll)
for CoregGP (T = 3, RBF, N = 16384 rows), MultiTaskGP in the Kronecker form (N = 4096 points, T = 4, L = 2, Matern: 16384
rows) and ExactGP (N = 16384).  Median and minimum over `--reps` runs after one warm-up.  Then, in runs of their own,
torch.profiler's per-kernel device time of one one-draw posterior and one MLL call per case: gram_lcm_kernel (and the
bytes it writes per second), mll_lcm_grad_kernel, mll_lcm_finish_kernel, and ExactGP's gram / mll_grad kernels.
Records the card's name, power limit and SM clock in the same process."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpax_b200  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")])) if out else {}


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()                      # every entry point returns after its device work has completed
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": float(np.median(ts)), "min_ms": float(np.min(ts))}


KERNELS = ("gram_lcm_kernel", "mll_lcm_grad_kernel", "mll_lcm_finish_kernel", "gram_fast_kernel", "gram_kernel",
           "mll_grad_kernel", "mll_finish_kernel")


def kernel_times(fn):
    """torch.profiler device time (ms, summed over launches) of the library's kernels named in KERNELS during fn()"""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type != DeviceType.CUDA:
            continue
        base = e.name.split("(")[0].split("<")[0].replace("void ", "").strip()
        if base in KERNELS:
            out[base] = out.get(base, 0.0) + e.device_time_total / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rows", type=int, default=16384)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    ctx = gpax_b200.default_context()
    n_rows, P, S, d = a.rows, 512, 8, 2
    res = {"card": card(), "rows": n_rows, "P": P, "S": S}

    def mt_case(T, L, group, kind):
        npts = n_rows // group
        X = rng.uniform(0, 4, (npts, d))
        Xn = rng.uniform(0, 4, (P // group, d))
        if group > 1:
            Xd, tt = np.repeat(X, T, 0), np.tile(np.arange(T), npts)
            Xnd, tn = np.repeat(Xn, T, 0), np.tile(np.arange(T), len(Xn))
        else:
            Xd, tt, Xnd, tn = X, rng.integers(0, T, npts), Xn, rng.integers(0, T, len(Xn))
        y = rng.standard_normal(len(Xd))
        th = np.concatenate([rng.uniform(0.5, 1.0, (S, L, d)), np.ones((S, L, 2))], -1)
        W = rng.normal(0, 0.7, (S, L, T, max(T - 1, 1)))
        B = np.einsum("sltr,slur->sltu", W, W) + 0.5 * np.eye(T)
        nz = np.full((S, T), 0.1)
        post = timed(lambda: ctx.posterior_multitask(kind, Xd, tt, y, Xnd, tn, th, B, nz, group, want=("mean", "var")), a.reps)
        mll = timed(lambda: ctx.mll_multitask(kind, Xd, tt, y, th[0], B[0], nz[0], group), a.reps)
        kp = kernel_times(lambda: ctx.posterior_multitask(kind, Xd, tt, y, Xnd, tn, th[:1], B[:1], nz[:1], group, want=("mean", "var")))
        km = kernel_times(lambda: ctx.mll_multitask(kind, Xd, tt, y, th[0], B[0], nz[0], group))
        # the LCM Gram of one posterior draw writes k_XX's lower triangle, k_pX and the P-vector of the prior variance
        nbytes = 8.0 * len(Xd) * (len(Xd) + 1) / 2 + 8.0 * len(Xd) * len(Xnd) + 8.0 * len(Xnd)
        return {"posterior": post, "mll": mll, "profile_posterior_ms": kp, "profile_mll_ms": km,
                "gram_lcm_bytes_per_s": nbytes / (kp["gram_lcm_kernel"] * 1e-3)}

    res["coreggp_T3_rbf"] = mt_case(3, 1, 1, "RBF")
    res["multitaskgp_kron_T4_L2_matern"] = mt_case(4, 2, 4, "Matern")
    X = rng.uniform(0, 4, (n_rows, d))
    Xn = rng.uniform(0, 4, (P, d))
    y = rng.standard_normal(n_rows)
    th = np.tile([0.7, 0.8, 1.0, 0.1, 1.0], (S, 1))
    res["exactgp_rbf"] = {"posterior": timed(lambda: ctx.posterior("RBF", X, y, Xn, th, want=("mean", "var")), a.reps),
                          "mll": timed(lambda: ctx.mll("RBF", X, y, th[0]), a.reps),
                          "profile_mll_ms": kernel_times(lambda: ctx.mll("RBF", X, y, th[0]))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
