"""ibnn_time.py -- time the NNGP likelihood step and the iBNN posterior, and print one JSON line.

  mll       median and minimum wall time of one b2gp_mll value + gradient call (it returns after its device work) over
            `--reps` runs after one warm-up, for the NNGP erf and ReLU kernels at depth 3 and for RBF on the same X (d <= 16
            only: b2gp_mll's RBF limit); N in {2048, 8192, 16384} x d in {3, 64}
  profile   in runs of their own, torch.profiler's device time of nngp_self_kernel, mll_nngp_grad_kernel and the NNGP
            gram_kernel launch in the likelihood step, and the share of the step's kernel time mll_nngp_grad_kernel takes
  predict   iBNN.predict with 8 draws (n = 1 sample each) at N = 16384, P = 1024, d = 3 (mean and samples), and one
            vi_iBNN.predict (mean and variance) on the same data with the device time of nngp_diag_kernel in it
Records the card's name, power limit and SM clock in the same process."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpax_b200  # noqa: E402
from tools.dkl_time import card, kernel_times, timed  # noqa: E402

NNGP = ("nngp_self_kernel", "mll_nngp_grad_kernel", "gram_kernel")
MLL_MAX_D = 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rows", default="2048,8192,16384")
    ap.add_argument("--dims", default="3,64")
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    ctx = gpax_b200.default_context()
    rng = np.random.default_rng(0)
    depth, p = 3, {"var_b": 0.6, "var_w": 1.7, "noise": 0.05}
    res = {"card": card(), "depth": depth, "cases": []}
    for N in [int(v) for v in a.rows.split(",")]:
        for d in [int(v) for v in a.dims.split(",")]:
            X = rng.uniform(-1, 1, (N, d))
            y = np.sin(3 * X[:, 0]) + 0.1 * rng.standard_normal(N)
            case = {"N": N, "d": d}
            th_nngp = np.r_[np.full(d, float(depth)), p["var_w"], p["noise"], p["var_b"]]
            th_rbf = np.r_[np.full(d, 0.8), 1.0, p["noise"], 1.0]
            runs = [("erf", "NNGP_erf", th_nngp), ("relu", "NNGP_relu", th_nngp)]
            if d <= MLL_MAX_D:                                  # b2gp_mll takes RBF up to d = 16 (its per-feature accumulators)
                runs.append(("rbf", "RBF", th_rbf))
            for name, kind, th in runs:
                step = lambda: ctx.mll(kind, X, y, th)          # noqa: E731
                case[name] = timed(step, a.reps)
                if not a.no_profile:
                    kt = kernel_times(step)
                    total = sum(kt.values())
                    prof = {"total_kernel_ms": total}
                    if kind != "RBF":
                        prof.update({k + "_ms": kt.get(k, 0.0) for k in NNGP})
                        prof["mll_nngp_grad_share"] = kt.get("mll_nngp_grad_kernel", 0.0) / total if total else None
                    case[name]["profile"] = prof
            res["cases"].append(case)
    N, P, S, d = 16384, 1024, 8, 3
    X = rng.uniform(-1, 1, (N, d))
    y = np.sin(3 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    Xn = rng.uniform(-1, 1, (P, d))
    m = gpax_b200.iBNN(d, depth=depth, activation="erf", ctx=ctx)
    m.X_train, m.y_train = X, y
    samples = {k: np.full(S, v) * (1 + 0.05 * np.arange(S)) for k, v in p.items()}
    pred = lambda: m.predict(0, Xn, samples, n=1)              # noqa: E731
    res["predict"] = {"N": N, "P": P, "draws": S, "d": d, **timed(pred, max(1, a.reps // 2))}
    if not a.no_profile:
        kt = kernel_times(pred)
        res["predict"]["profile"] = {"gram_kernel_ms": kt.get("gram_kernel", 0.0), "total_kernel_ms": sum(kt.values())}
    v = gpax_b200.vi_iBNN(d, depth=depth, activation="erf", ctx=ctx)
    v.X_train, v.y_train = X, y
    vpred = lambda: v.predict(0, Xn, p)                       # noqa: E731
    res["vi_predict"] = {"N": N, "P": P, "d": d, **timed(vpred, a.reps)}
    if not a.no_profile:
        kt = kernel_times(vpred)
        res["vi_predict"]["profile"] = {"nngp_diag_kernel_ms": kt.get("nngp_diag_kernel", 0.0), "total_kernel_ms": sum(kt.values())}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
