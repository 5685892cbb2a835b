"""callable_time.py -- time the user-kernel-callable route against the fused RBF route, and print one JSON line.

  loglik    one log-joint evaluation (value + gradient) of an ExactGP on a NumPy RBF callable (GramLogJoint) at
            N in {1024, 4096} x d in {1, 8} ARD (p = 3 and 10 differenced coordinates): wall time, the host time spent
            inside the callable (K and the 2p finite-difference evaluations), the device time of the b2gp_mll_gram call
            (b2gp_timing total_ms), and the same evaluation on the fused "RBF" LogJoint
  predict   ExactGP.predict with S = 100 draws, n = 1, P = 1000, d = 1 on both routes (--predict-rows), with the host
            time inside the callable
Median and minimum over `--reps` runs after one warm-up.  Records the card's name, power limit and SM clock."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpax_b200  # noqa: E402
from gpax_b200.inference import LogJoint, make_log_joint  # noqa: E402
from tools.dkl_time import card, timed  # noqa: E402


class TimedRBF:
    """k(X, Z, params, noise, jitter) on NumPy, as a user would write it; accumulates the host time spent in it"""

    def __init__(self):
        self.ms = 0.0

    def __call__(self, X, Z, params, noise=0, jitter=1e-6, **kw):
        t0 = time.perf_counter()
        ell = np.asarray(params["k_length"], dtype=np.float64).reshape(-1)
        A, B = X / ell, Z / ell
        r2 = (A * A).sum(1)[:, None] - 2.0 * A @ B.T + (B * B).sum(1)[None, :]
        k = float(params["k_scale"]) * np.exp(-0.5 * np.maximum(r2, 0.0))
        if X.shape == Z.shape:
            k[np.diag_indices(X.shape[0])] += noise + jitter
        self.ms += (time.perf_counter() - t0) * 1e3
        return k


def models(N, d, rng, ctx):
    X = rng.uniform(0, 1, (N, d))
    y = np.sin(4 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    k = TimedRBF()
    mc, mf = gpax_b200.ExactGP(d, k, ctx=ctx), gpax_b200.ExactGP(d, "RBF", ctx=ctx)
    for m in (mc, mf):
        m.X_train, m.y_train = X, y
    return mc, mf, k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rows", default="1024,4096")
    ap.add_argument("--dims", default="1,8")
    ap.add_argument("--predict-rows", default="1024,4096")
    ap.add_argument("--draws", type=int, default=100)
    ap.add_argument("--test-points", type=int, default=1000)
    a = ap.parse_args()
    ctx = gpax_b200.default_context()
    rng = np.random.default_rng(0)
    res = {"card": card(), "loglik": [], "predict": []}
    for N in [int(v) for v in a.rows.split(",")]:
        for d in [int(v) for v in a.dims.split(",")]:
            mc, mf, k = models(N, d, rng, ctx)
            lc, lf = make_log_joint(mc), LogJoint(mf)
            u = lf.init_u()
            dev = []

            def eval_callable():
                lc(u, True)
                dev.append(ctx.last_timing()["total_ms"])
            k.ms = 0.0
            t = timed(eval_callable, a.reps)
            host = k.ms / (a.reps + 1)
            res["loglik"].append({"N": N, "d": d, "p": lc.dim, "callable": t, "callable_host_kernel_ms": host,
                                  "mll_gram_device_ms": float(np.median(dev)), "fused": timed(lambda: lf(u, True), a.reps)})
            print(json.dumps(res["loglik"][-1]), file=sys.stderr)
    S, P = a.draws, a.test_points
    for N in [int(v) for v in a.predict_rows.split(",")]:
        mc, mf, k = models(N, 1, rng, ctx)
        Xt = np.linspace(0, 1, P)
        samples = {"k_length": rng.uniform(0.2, 0.5, (S, 1)), "k_scale": rng.uniform(0.8, 1.5, S), "noise": rng.uniform(0.05, 0.2, S)}
        reps = max(1, a.reps // 2)
        k.ms = 0.0
        tc = timed(lambda: mc.predict(0, Xt, samples, n=1), reps)
        host = k.ms / (reps + 1)
        tf = timed(lambda: mf.predict(0, Xt, samples, n=1), reps)
        res["predict"].append({"N": N, "S": S, "P": P, "callable": tc, "callable_host_kernel_ms": host, "fused": tf})
        print(json.dumps(res["predict"][-1]), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
