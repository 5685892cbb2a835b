"""Crossover of the fp64 tall-panel route against the recursive one (the `tall_min_fp64` default, DESIGN.md 4.2).

  python tools/tall_fp64_crossover.py [--reps 3] [--out DIR]

For N in 4096, 8192, 12288, 16384 (bench.py's inputs otherwise: d = 3, P = 1024, RBF, seeded draws), times one posterior
step -- 8 draws on 8 streams, and one draw on one stream -- with panel = 0 (recursive: potrf_rec, then trsm_rec of the
test-point rows) and panel = 1024 (tall-panel route, tall_min_fp64 lowered to 4096), the same command alternating the two
values.  Device time per step from the library's CUDA events (b2gp_last_timing total_ms).  Writes DIR/crossover.json.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=".", help="output directory (default: the current directory)")
    args = ap.parse_args()
    from gpax_b200 import _ffi as ffi
    ctx = ffi.Context(0)
    ctx.set_option("tall_min_fp64", 4096)
    d, P = 3, 1024
    res = []
    for N in (4096, 8192, 12288, 16384):
        rng = np.random.default_rng(4)
        X = rng.uniform(0, 1, (N, d))
        y = np.sin(3 * X[:, 0]) * np.cos(2 * X[:, 1]) + X[:, 2] + 0.1 * rng.standard_normal(N)
        Xn = rng.uniform(0, 1, (P, d))
        for S, streams in ((8, 8), (1, 1)):
            theta = np.empty((S, d + 3))
            theta[:, :d] = 0.3 * np.exp(0.05 * rng.standard_normal((S, d)))
            theta[:, d], theta[:, d + 1], theta[:, d + 2] = 1.0, 0.1, 1.0
            ctx.set_option("streams", streams)
            dX, dy, dXn, dth = ctx.to_device(X), ctx.to_device(y), ctx.to_device(Xn), ctx.to_device(theta)
            dmean, dvar = ctx.alloc((S, P)), ctx.alloc((S, P))
            info = np.zeros(S, dtype=np.int32)

            def step():
                ctx._check(ctx.lib.b2gp_posterior(ctx.h, ffi.KIND["RBF"], dX.ptr, N, dy.ptr, 0, dXn.ptr, P, d, S, dth.ptr, 0, 1e-6,
                                                  ffi.OUT_MEAN | ffi.OUT_VAR | ffi.FLAG_DEVICE_PTRS, dmean.ptr, dvar.ptr, None, None,
                                                  0, None, info.ctypes.data, None))
                assert (info == 0).all(), info
                return ctx.last_timing()["total_ms"]

            ms = {0: [], 1024: []}
            for panel in (0, 1024):                      # warm-up of both routes
                ctx.set_option("panel", panel)
                step()
            for _ in range(args.reps):
                for panel in (0, 1024):
                    ctx.set_option("panel", panel)
                    ms[panel].append(step())
            row = {"N": N, "draws": S, "streams": streams, "ms_panel0": ms[0], "ms_panel1024": ms[1024],
                   "speedup": float(np.median(ms[0]) / np.median(ms[1024]))}
            res.append(row)
            print(json.dumps(row), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "crossover.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
