"""Time optimize_acq on MultiTaskGP with the closed-form gradient (b2gp_posterior_multitask_grad) against SciPy's finite
differences (d + 1 acq_fn calls per gradient, d counting the task column), on hand-set draws.  T = 2 tasks, L = 2
latents, the multitask form with the task column fixed by its bounds, EI over n = 8 predictive samples per draw (at S = 1
a single sample would have no spread).  Per configuration (N GP rows, d data features, S draws):

  analytic_eval_ms   median wall time of one evaluation of the analytic objective (value and gradient together)
  fd_grad_ms         median wall time of one finite-difference gradient: d + 2 acq_fn calls (the value and one call per
                     column, the fixed task column included, as L-BFGS-B's differences take them)
  opt_analytic_s     one whole optimize_acq(EI) run on the analytic route, its posterior calls and the EI it reached
  opt_fd_s           the same run with the analytic route switched off (what optimize_acq did before it existed); not
                     run (null) where one finite-difference gradient takes longer than --fd-budget-ms

and, in a run of its own under torch.profiler, gram_dx_lcm_kernel's device time and the bytes it writes.  The card's
name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; needs a GPU.

    python tools/mtgp_acq_time.py [--reps 3] [--guesses 16] [--fd-budget-ms 1500] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T, L = 2, 2
KW = {"n": 8}


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


class _Draws:
    def __init__(self, samples):
        self.samples = samples

    def get_samples(self, group_by_chain=False):
        return self.samples


def make_mtgp(ctx, N, d, S):
    from gpax_b200 import MultiTaskGP
    rng = np.random.default_rng(N + d + S)
    Xd = rng.uniform(-1, 1, (N, d))
    t = np.arange(N) % T
    y = np.sin(3 * Xd[:, 0]) + np.cos(2 * Xd[:, -1]) + 0.3 * t + 0.05 * rng.standard_normal(N)
    m = MultiTaskGP(d, "RBF", num_latents=L, num_tasks=T, ctx=ctx)
    m.X_train, m.y_train = np.c_[Xd, t], y
    m.mcmc = _Draws({"k_length": rng.uniform(0.5, 1.0, (S, L, d)) * np.sqrt(d), "k_scale": rng.uniform(0.8, 1.5, (S, L)),
                     "W": rng.normal(0, 0.7, (S, L, T, 1)), "v": rng.uniform(0.3, 0.8, (S, L, T)),
                     "noise": rng.uniform(0.01, 0.05, (S, T))})
    return m


def median_ms(fn, reps):
    fn()                                            # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()                                        # returns host values: every call ends in a device synchronise
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def measure(model, d, reps, guesses, fd_budget_ms):
    from gpax_b200 import acquisition as acq, prng
    key = prng.PRNGKey(3)
    D = d + 1                                        # the data columns and the task column
    lb, ub = [-1.0] * d + [1.0], [1.0] * d + [1.0]
    x = np.r_[np.full(d, 0.1), 1.0]
    f = acq._analytic_objective("EI", key, model, D, KW)
    out = {"analytic_eval_ms": median_ms(lambda: f(x), reps)}

    def fd_grad():
        base = acq.EI(key, model, x[None], **KW)
        for k in range(D):
            e = np.zeros(D)
            e[k] = 1.4901161193847656e-08
            acq.EI(key, model, (x + e)[None], **KW)
        return base
    out["fd_grad_ms"] = median_ms(fd_grad, 1)

    ctx = model.ctx
    for route in ("analytic", "fd"):
        if route == "fd" and out["fd_grad_ms"] > fd_budget_ms:
            out.update({"opt_fd_s": None, "opt_fd_calls": None, "opt_fd_ei": None})
            continue
        calls = {"posterior_multitask": 0, "posterior_multitask_grad": 0}
        for name in calls:                          # count the library calls through instance attributes
            bound = getattr(ctx, name)

            def wrapped(*a, _fn=bound, _name=name, **k):
                calls[_name] += 1
                return _fn(*a, **k)
            setattr(ctx, name, wrapped)
        orig = acq._analytic_kind
        if route == "fd":
            acq._analytic_kind = lambda *a, **k: None
        try:
            t0 = time.perf_counter()
            xo = acq.optimize_acq(key, model, acq.EI, guesses, lb, ub, **KW)
            sec = time.perf_counter() - t0
        finally:
            acq._analytic_kind = orig
            del ctx.posterior_multitask, ctx.posterior_multitask_grad
        ei = float(np.asarray(acq.EI(key, model, np.asarray(xo, np.float64).reshape(1, D), **KW)).reshape(-1)[0])
        out[f"opt_{route}_s"] = sec
        out[f"opt_{route}_calls"] = calls
        out[f"opt_{route}_ei"] = ei
    return out


def dx_kernel_time(ctx, N, P, d, reps=5):
    """gram_dx_lcm_kernel's device time from torch.profiler (a run of its own) and the bytes it writes, 8 P d N"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(N + P + d)
    X, Xn = rng.uniform(-1, 1, (N, d)), rng.uniform(-1, 1, (P, d))
    tt, tn = np.arange(N) % T, np.arange(P) % T
    y = rng.standard_normal(N)
    theta = np.concatenate([np.full((1, L, d), 0.8 * np.sqrt(d)), np.ones((1, L, 2))], axis=2)
    B = np.tile(np.eye(T) + 0.3, (1, L, 1, 1))
    noise = np.full((1, T), 0.02)
    run = lambda: ctx.posterior_multitask_grad("RBF", X, tt, y, Xn, tn, theta, B, noise, want=("dmean",))   # noqa: E731
    run()                                                                                                   # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            run()
        torch.cuda.synchronize()
    us = [getattr(e, "device_time", None) or e.cuda_time for e in prof.events() if "gram_dx_lcm_kernel" in e.name]
    if not us:
        raise RuntimeError("torch.profiler recorded no gram_dx_lcm_kernel")
    nbytes = 8.0 * P * d * N
    return {"N": N, "P": P, "d": d, "L": L, "T": T, "kernel_us": float(np.median(us)), "bytes_written": nbytes,
            "GB_per_s": nbytes / (float(np.median(us)) * 1e-6) / 1e9, "launches_seen": len(us)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--guesses", type=int, default=16)
    ap.add_argument("--fd-budget-ms", type=float, default=1500.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import scipy.optimize  # noqa: F401  (imported by optimize_acq; its first import would land in the first timed run)
    from gpax_b200 import _ffi
    ctx = _ffi.Context(0)
    res = {"gpu": gpu_info(), "acq": "EI", "n": KW["n"], "T": T, "L": L, "rows": []}
    for N in (256, 2048, 8192):
        for d in (1, 4, 16):
            for S in (1, 64):
                row = {"model": "MultiTaskGP", "N": N, "d": d, "S": S}
                row.update(measure(make_mtgp(ctx, N, d, S), d, a.reps, a.guesses, a.fd_budget_ms))
                res["rows"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
    res["dx_kernel"] = [dx_kernel_time(ctx, N, P, d) for N, P, d in ((8192, 1, 16), (8192, 256, 4), (8192, 256, 16))]
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
