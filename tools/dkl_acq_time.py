"""Time optimize_acq on viDKL and DKL with the closed-form gradient (b2gp_dkl_posterior_grad) against SciPy's finite
differences (D + 1 acq_fn calls per gradient), on hand-set weights and draws.  Per configuration:

  analytic_eval_ms   median wall time of one evaluation of the analytic objective (value and gradient together; for
                     viDKL the factor of the training embedding is cached after the first one)
  fd_grad_ms         median wall time of one finite-difference gradient: D + 1 acq_fn calls
  opt_analytic_s     one whole optimize_acq(EI) run on the analytic route, its evaluations and the EI it reached
  opt_fd_s           the same run with the analytic route switched off (what optimize_acq did before it existed)

and, in runs of their own under torch.profiler, mlp_input_vjp_kernel's device time and the weight bytes it reads.  The
card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; needs a GPU.

    python tools/dkl_acq_time.py [--reps 5] [--guesses 16] [--out result.json]
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


def flat_weights(rng, D, widths, S, scale=1.0):
    parts, i = [], D
    for w in widths:
        parts.append((rng.standard_normal((S, i * w)) * scale / np.sqrt(i), 0.1 * rng.standard_normal((S, w))))
        i = w
    return np.concatenate([np.concatenate([W, b], axis=1) for W, b in parts], axis=1)


def make_vidkl(ctx, N, D):
    from gpax_b200 import viDKL
    rng = np.random.default_rng(N + D)
    X = rng.uniform(-1, 1, (N, D))
    y = np.sin(3 * X[:, 0]) + np.cos(2 * X[:, -1]) + 0.05 * rng.standard_normal(N)
    m = viDKL(D, 2, "RBF", ctx=ctx)
    m.X_train, m.y_train = X, y
    m.nn_params = m.from_flat(flat_weights(rng, D, m.widths, 1)[0])
    m.kernel_params = {"k_length": np.array([0.8, 1.1]), "k_scale": np.array(1.2), "noise": np.array(0.02)}
    return m


class _Draws:
    def __init__(self, samples):
        self.samples = samples

    def get_samples(self, group_by_chain=False):
        return self.samples


def make_dkl(ctx, N, D, S):
    from gpax_b200 import DKL
    rng = np.random.default_rng(N + D + S)
    X = rng.uniform(-1, 1, (N, D))
    y = np.sin(3 * X[:, 0]) + np.cos(2 * X[:, -1]) + 0.05 * rng.standard_normal(N)
    m = DKL(D, 2, "RBF", ctx=ctx)
    m.X_train, m.y_train = X, y
    samples = m.from_flat(flat_weights(rng, D, m.widths, S))
    samples.update({"k_length": rng.uniform(0.7, 1.3, (S, 2)), "k_scale": rng.uniform(0.8, 1.5, S),
                    "noise": rng.uniform(0.01, 0.05, S)})
    m.mcmc = _Draws(samples)
    return m


def median_ms(fn, reps):
    fn()                                            # warm-up (and, for viDKL, the cached factor)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()                                        # returns host values: every call ends in a device synchronise
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def measure(model, D, reps, guesses):
    from gpax_b200 import acquisition as acq, prng
    key = prng.PRNGKey(3)
    lb, ub = [-1.0] * D, [1.0] * D
    x = np.full(D, 0.1)
    f = acq._analytic_objective("EI", key, model, D, {})
    out = {"analytic_eval_ms": median_ms(lambda: f(x), reps)}

    def fd_grad():
        base = acq.EI(key, model, x[None])
        for k in range(D):
            e = np.zeros(D)
            e[k] = 1.4901161193847656e-08
            acq.EI(key, model, (x + e)[None])
        return base
    out["fd_grad_ms"] = median_ms(fd_grad, max(1, reps // 2))

    for route in ("analytic", "fd"):
        calls = {"predict": 0, "posterior_grad": 0}
        for name in calls:                          # count the posterior calls through instance attributes
            bound = getattr(model, name if name == "predict" else "_posterior_grad")

            def wrapped(*a, _fn=bound, _name=name, **k):
                calls[_name] += 1
                return _fn(*a, **k)
            setattr(model, name if name == "predict" else "_posterior_grad", wrapped)
        orig = acq._analytic_kind
        if route == "fd":
            acq._analytic_kind = lambda *a, **k: None
        try:
            t0 = time.perf_counter()
            xo = acq.optimize_acq(key, model, acq.EI, guesses, lb, ub)
            sec = time.perf_counter() - t0
        finally:
            acq._analytic_kind = orig
            del model.predict, model._posterior_grad
        ei = float(np.asarray(acq.EI(key, model, np.asarray(xo, np.float64).reshape(1, D))).reshape(-1)[0])
        out[f"opt_{route}_s"] = sec
        out[f"opt_{route}_calls"] = calls
        out[f"opt_{route}_ei"] = ei
    return out


def vjp_kernel_time(ctx, D, S, P, widths=(64, 64, 2), reps=5):
    """mlp_input_vjp_kernel's device time from torch.profiler (a run of its own) and the weight bytes it reads per launch
    (every weight set's W_l once per CTA row of the bottom-layer tiling, upper layers once per tile)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(D)
    X, Xn = rng.uniform(-1, 1, (64, D)), rng.uniform(-1, 1, (P, D))
    y = rng.standard_normal(64)
    flats = flat_weights(rng, D, widths, S)
    theta = np.tile([0.8, 1.1, 1.2, 0.02, 1.0], (S, 1))
    ctx.dkl_posterior_grad("RBF", X, y, Xn, list(widths), 0, flats, theta)       # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.dkl_posterior_grad("RBF", X, y, Xn, list(widths), 0, flats, theta)
        torch.cuda.synchronize()
    us = [getattr(e, "device_time", None) or e.cuda_time for e in prof.events() if "mlp_input_vjp_kernel" in e.name]
    if not us:
        raise RuntimeError("torch.profiler recorded no mlp_input_vjp_kernel")
    tiles = -(-D // 64)
    upper = sum(a * b for a, b in zip(widths[:-1], widths[1:]))
    nbytes = 8.0 * S * P * (D * widths[0] + tiles * upper)
    return {"D": D, "S": S, "P": P, "widths": list(widths), "kernel_us": float(np.median(us)), "weight_bytes": nbytes,
            "GB_per_s": nbytes / (float(np.median(us)) * 1e-6) / 1e9, "launches_seen": len(us)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--guesses", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import scipy.optimize  # noqa: F401  (imported by optimize_acq; its first import would land in the first timed run)
    from gpax_b200 import _ffi
    ctx = _ffi.Context(0)
    res = {"gpu": gpu_info(), "acq": "EI", "rows": []}
    for N in (500, 2000, 8000):
        for D in (4, 64):
            row = {"model": "viDKL", "N": N, "D": D, "z_dim": 2}
            row.update(measure(make_vidkl(ctx, N, D), D, a.reps, a.guesses))
            res["rows"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    for S in (50, 200):
        row = {"model": "DKL", "S": S, "N": 200, "D": 6, "z_dim": 2, "hidden": [64, 32]}
        row.update(measure(make_dkl(ctx, 200, 6, S), 6, a.reps, a.guesses))
        res["rows"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    res["vjp_kernel"] = [vjp_kernel_time(ctx, D, S, P) for D, S, P in ((64, 1, 1), (4096, 1, 1), (4096, 1, 64), (6, 200, 1))]
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
