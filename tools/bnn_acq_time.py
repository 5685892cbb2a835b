"""Time optimize_acq on a BNN with the closed-form gradient (b2gp_bnn_predict_grad, weight sets resident on the device)
against SciPy's finite differences (D + 1 acq_fn calls per gradient, each a b2gp_bnn_predict call that uploads every
weight set), for the default [64, 32] network with hand-set draws.  Per configuration (D, S):

  analytic_eval_ms        median wall time of one evaluation of the analytic objective (value and gradient together)
  launches_per_eval       kernel launches of that evaluation's library call
  fd_grad_ms              median wall time of one finite-difference gradient: D + 1 EI calls
  opt_analytic_s          one whole optimize_acq(EI) run on the analytic route, its library calls and the EI it reached
  opt_fd_s                the same run with the analytic route switched off, for S <= --fd-run-max-s only: every EI
                          call draws the S-draw normal stream on the host (about 1.3 s at S = 8000 on one CPU core), so
                          a whole finite-difference run there takes minutes of host time and says nothing new

and, in a run of its own under torch.profiler, bnn_predict_grad_kernel's device time.  The card's name, power limit and
maximum SM clock are read in the same run.  Prints one JSON line; needs a GPU.

    python tools/bnn_acq_time.py [--reps 7] [--guesses 16] [--fd-run-max-s 2000] [--out result.json]
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


class _Draws:
    def __init__(self, samples):
        self.samples = samples

    def get_samples(self, group_by_chain=False):
        return self.samples


def make_bnn(ctx, D, S):
    """a BNN with S hand-set draws around one smooth network (weights scaled per draw), noise 0.05-0.15"""
    from gpax_b200 import BNN
    m = BNN(D, 1, ctx=ctx)
    rng = np.random.default_rng(D + S)
    parts, i = [], D
    for w in m.widths:
        W = rng.standard_normal((i, w)) / np.sqrt(i)
        parts.append(np.concatenate([W.reshape(-1), 0.1 * rng.standard_normal(w)]))
        i = w
    flat = np.concatenate(parts)[None] * rng.uniform(0.8, 1.2, (S, 1))
    samples = m.from_flat(flat)
    samples["noise"] = rng.uniform(0.05, 0.15, S)
    m.X_train = rng.uniform(-1, 1, (32, D))
    m.y_train = np.zeros((32, 1))
    m.mcmc = _Draws(samples)
    return m


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()                                        # returns host values: every call ends in a device synchronise
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def measure(ctx, model, D, reps, guesses, fd_run):
    from gpax_b200 import acquisition as acq, prng
    key = prng.PRNGKey(3)
    lb, ub = [-1.0] * D, [1.0] * D
    x = np.full(D, 0.1)
    out = {}
    with acq._bnn_objective("EI", key, model, D, {}) as f:
        out["analytic_eval_ms"] = median_ms(lambda: f(x), reps)
        f(x)
        out["launches_per_eval"] = ctx.last_timing()["launches"]

    def fd_grad():
        base = acq.EI(key, model, x[None])
        for k in range(D):
            e = np.zeros(D)
            e[k] = 1.4901161193847656e-08
            acq.EI(key, model, (x + e)[None])
        return base
    out["fd_grad_ms"] = median_ms(fd_grad, max(1, reps // 2))

    for route in ("analytic", "fd") if fd_run else ("analytic",):
        calls = {"bnn_predict": 0, "bnn_predict_grad": 0}
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
            xo = acq.optimize_acq(key, model, acq.EI, guesses, lb, ub)
            sec = time.perf_counter() - t0
        finally:
            acq._analytic_kind = orig
            del ctx.bnn_predict, ctx.bnn_predict_grad
        ei = float(np.asarray(acq.EI(key, model, np.asarray(xo, np.float64).reshape(1, D))).reshape(-1)[0])
        out[f"opt_{route}_s"] = sec
        out[f"opt_{route}_calls"] = calls
        out[f"opt_{route}_ei"] = ei
    return out


def kernel_time(ctx, D, S, reps=20):
    """bnn_predict_grad_kernel's device time at one point from torch.profiler (a run of its own), weight sets resident"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    m = make_bnn(ctx, D, S)
    flat = np.atleast_2d(m.to_flat(m.get_samples()))
    Pd, Xd = ctx.to_device(flat), ctx.to_device(np.full((1, D), 0.1))
    try:
        ctx.bnn_predict_grad(Xd, m.widths, 1, Pd)                   # warm-up
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                ctx.bnn_predict_grad(Xd, m.widths, 1, Pd)
            torch.cuda.synchronize()
    finally:
        Pd.free()
        Xd.free()
    us = [getattr(e, "device_time", None) or e.cuda_time for e in prof.events() if "bnn_predict_grad_kernel" in e.name]
    if not us:
        raise RuntimeError("torch.profiler recorded no bnn_predict_grad_kernel")
    nbytes = 8.0 * flat.size
    med = float(np.median(us))
    return {"D": D, "S": S, "P": 1, "kernel_us": med, "weight_bytes": nbytes, "GB_per_s": nbytes / (med * 1e-6) / 1e9,
            "launches_seen": len(us)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--guesses", type=int, default=16)
    ap.add_argument("--fd-run-max-s", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import scipy.optimize  # noqa: F401  (imported by optimize_acq; its first import would land in the first timed run)
    from gpax_b200 import _ffi
    ctx = _ffi.Context(0)
    res = {"gpu": gpu_info(), "acq": "EI", "hidden": [64, 32], "rows": []}
    for D in (1, 4):
        for S in (100, 2000, 8000):
            row = {"D": D, "S": S}
            row.update(measure(ctx, make_bnn(ctx, D, S), D, a.reps, a.guesses, S <= a.fd_run_max_s))
            res["rows"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    res["kernel"] = [kernel_time(ctx, D, S) for D in (1, 4) for S in (100, 2000, 8000)]
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
