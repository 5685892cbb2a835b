"""sparse_callable_time.py -- time viSparseGP on a user kernel callable against the fused RBF route, print a table and
one JSON line.

  loglik    one log-joint evaluation (value + gradient w.r.t. the sites and Xu) of viSparseGP on a NumPy RBF callable
            (SparseGramLogJoint: 3 differenced kernel coordinates at d = 2, 2 d shifted Kuf and 4 d shifted Kuu calls
            for Xu) at N in {16384, 65536} x M in {256, 1024}: wall time, the host time inside the callable, the device
            time of the b2gp_sparse_elbo_gram call (b2gp_timing total_ms), and the same evaluation on the fused "RBF"
            SparseLogJoint
  predict   viSparseGP.predict at P = 4096 on both routes, with the host time inside the callable
Median and minimum over `--reps` runs after one warm-up.  Records the card's name, power limit and SM clock."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpax_b200  # noqa: E402
from gpax_b200.inference import SparseGramLogJoint, SparseLogJoint  # noqa: E402
from tools.callable_time import TimedRBF  # noqa: E402
from tools.dkl_time import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rows", default="16384,65536")
    ap.add_argument("--inducing", default="256,1024")
    ap.add_argument("--test-points", type=int, default=4096)
    a = ap.parse_args()
    ctx = gpax_b200.default_context()
    rng = np.random.default_rng(0)
    d, P = 2, a.test_points
    res = {"card": card(), "loglik": [], "predict": []}
    for N in [int(v) for v in a.rows.split(",")]:
        X = rng.uniform(0, 1, (N, d))
        y = np.sin(4 * X[:, 0]) * np.cos(3 * X[:, 1]) + 0.1 * rng.standard_normal(N)
        Xs = rng.uniform(0, 1, (P, d))
        for M in [int(v) for v in a.inducing.split(",")]:
            Xu = X[rng.choice(N, M, replace=False)]
            k = TimedRBF()
            mc, mf = gpax_b200.viSparseGP(d, k, ctx=ctx), gpax_b200.viSparseGP(d, "RBF", ctx=ctx)
            for m in (mc, mf):
                m.X_train, m.y_train, m.Xu = X, y, Xu
            lc, lf = SparseGramLogJoint(mc, Xu), SparseLogJoint(mf, Xu)
            u = lf.init_u()
            dev = []

            def eval_callable():
                lc(u, False)
                dev.append(ctx.last_timing()["total_ms"])
            k.ms = 0.0
            t = timed(eval_callable, a.reps)
            row = {"N": N, "M": M, "callable": t, "callable_host_kernel_ms": k.ms / (a.reps + 1),
                   "elbo_gram_device_ms": float(np.median(dev)), "fused": timed(lambda: lf(u, False), a.reps)}
            res["loglik"].append(row)
            print(json.dumps(row), file=sys.stderr)
            params = {"k_length": np.full(d, 0.3), "k_scale": 1.0, "noise": 0.05}
            k.ms = 0.0
            tc = timed(lambda: mc.predict(0, Xs, params), a.reps)
            row = {"N": N, "M": M, "P": P, "callable": tc, "callable_host_kernel_ms": k.ms / (a.reps + 1),
                   "fused": timed(lambda: mf.predict(0, Xs, params), a.reps)}
            res["predict"].append(row)
            print(json.dumps(row), file=sys.stderr)
    print(f"card: {res['card']}")
    print("log joint + gradient (ms, median)        callable  in callable  device (elbo_gram)  fused")
    for r in res["loglik"]:
        print(f"  N={r['N']:6d} M={r['M']:5d}              {r['callable']['median_ms']:10.1f} {r['callable_host_kernel_ms']:11.1f}"
              f" {r['elbo_gram_device_ms']:19.1f} {r['fused']['median_ms']:6.1f}")
    print(f"predict at P={P} (ms, median)            callable  in callable  fused")
    for r in res["predict"]:
        print(f"  N={r['N']:6d} M={r['M']:5d}              {r['callable']['median_ms']:10.1f} {r['callable_host_kernel_ms']:11.1f}"
              f" {r['fused']['median_ms']:6.1f}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
