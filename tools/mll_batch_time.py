"""mll_batch_time.py -- time b2gp_mll_batch against the single-member calls it replaces, and print one JSON line.

  calls   at (B, N) in {(1, 32), (1, 128), (16, 64), (132, 128), (8, 512), (2, 2048)}, RBF and Periodic, d in {1, 3}:
          one mll_batch call (value + gradient) against B ctx.mll calls (vExactGP's per-task likelihoods), and one
          mll_batch call with the input gradient against B ctx.dkl_mll(n_layers = 0) calls (UIGP's likelihood); host
          wall time per call and kernel launches per call (b2gp_timing)
  sweep   B = 1 at N in {16, 24, ..., 128}, every kind, d in {1, 3}: one mll_batch call against one ctx.mll call, and with
          the input gradient against one ctx.dkl_mll(n_layers = 0) call -- where the one-launch route stops winning for a
          single member (UIGP's case), which sets B2GP_MLL_BATCH_SMALL_MAX_N; the small-route column measures the
          one-launch route only up to the bound the library was built with
  fits    vExactGP.fit (B = 8, N = 64) and UIGP.fit (N = 64), 200 + 200 draws: wall time and gradient evaluations
Median and minimum over `--reps` runs after one warm-up.  Records the card's name, power limit and SM clock."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpax_b200  # noqa: E402
from tools.dkl_time import card, timed  # noqa: E402

SIZES = [(1, 32), (1, 128), (16, 64), (132, 128), (8, 512), (2, 2048)]


def problem(kind, B, N, d, rng):
    X = rng.uniform(0, 1, (B, N, d))
    y = np.sin(4 * X[..., 0]) + 0.1 * rng.standard_normal((B, N))
    th = np.concatenate([np.full((B, d), 0.3 * np.sqrt(d)), np.full((B, 1), 1.2), np.full((B, 1), 0.1),
                         np.full((B, 1), 0.8 if kind == "Periodic" else 1.0)], axis=1)
    return X, y, th


def calls(ctx, reps, rng):
    rows = []
    for kind in ("RBF", "Periodic"):
        for d in (1, 3):
            for B, N in SIZES:
                X, y, th = problem(kind, B, N, d, rng)
                r = {"kind": kind, "d": d, "B": B, "N": N}
                r["batch"] = timed(lambda: ctx.mll_batch(kind, X, y, th, 1e-6, True), reps)
                r["batch_launches"] = ctx.last_timing()["launches"]
                r["loop_mll"] = timed(lambda: [ctx.mll(kind, X[b], y[b], th[b], 1e-6) for b in range(B)], reps)
                r["mll_launches_per_member"] = ctx.last_timing()["launches"]
                r["batch_grad_x"] = timed(lambda: ctx.mll_batch(kind, X, y, th, 1e-6, True, False, True), reps)
                r["loop_dkl_mll"] = timed(lambda: [ctx.dkl_mll(kind, X[b], y[b], [], 0, np.zeros(0), th[b], 1e-6, want_params=False,
                                                               want_z=True) for b in range(B)], reps)
                r["speedup_vs_mll"] = r["loop_mll"]["median_ms"] / r["batch"]["median_ms"]
                r["speedup_vs_dkl_mll"] = r["loop_dkl_mll"]["median_ms"] / r["batch_grad_x"]["median_ms"]
                rows.append(r)
    return rows


SWEEP_N = [16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128]


def sweep(ctx, reps, rng):
    rows = []
    for kind in ("RBF", "Matern", "Periodic"):
        for d in (1, 3):
            for N in SWEEP_N:
                X, y, th = problem(kind, 1, N, d, rng)
                r = {"kind": kind, "d": d, "N": N}
                c0 = ctx.path_counts()["mll_batch_small"]
                r["batch"] = timed(lambda: ctx.mll_batch(kind, X, y, th, 1e-6, True), reps)
                r["small_route"] = ctx.path_counts()["mll_batch_small"] > c0
                r["mll"] = timed(lambda: ctx.mll(kind, X[0], y[0], th[0], 1e-6), reps)
                r["batch_grad_x"] = timed(lambda: ctx.mll_batch(kind, X, y, th, 1e-6, True, False, True), reps)
                r["dkl_mll"] = timed(lambda: ctx.dkl_mll(kind, X[0], y[0], [], 0, np.zeros(0), th[0], 1e-6, want_params=False,
                                                         want_z=True), reps)
                r["speedup_vs_mll"] = r["mll"]["median_ms"] / r["batch"]["median_ms"]
                r["speedup_vs_dkl_mll"] = r["dkl_mll"]["median_ms"] / r["batch_grad_x"]["median_ms"]
                rows.append(r)
    return rows


def fits(ctx, draws, rng):
    out = {}
    X = rng.uniform(0, 1, (8, 64, 1))
    y = np.sin(6 * X[..., 0]) + 0.05 * rng.standard_normal((8, 64))
    m = gpax_b200.vExactGP(1, "RBF", ctx=ctx)
    t0 = time.perf_counter()
    m.fit(0, X, y, num_warmup=draws, num_samples=draws, progress_bar=False, print_summary=False)
    out["vExactGP_B8_N64"] = {"wall_s": time.perf_counter() - t0, "grad_evals": m.mcmc.stats[0]["grad_evals"]}
    x = np.linspace(0, 1, 64)
    m = gpax_b200.UIGP(1, "RBF", ctx=ctx)
    t0 = time.perf_counter()
    m.fit(0, x, np.sin(6 * x) + 0.05 * rng.standard_normal(64), num_warmup=draws, num_samples=draws, progress_bar=False,
          print_summary=False)
    out["UIGP_N64"] = {"wall_s": time.perf_counter() - t0, "grad_evals": m.mcmc.stats[0]["grad_evals"]}
    for v in out.values():
        v["ms_per_eval"] = 1e3 * v["wall_s"] / v["grad_evals"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--draws", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = gpax_b200._ffi.Context(0)
    rng = np.random.default_rng(0)
    res = {"card": card(), "calls": calls(ctx, a.reps, rng), "sweep": sweep(ctx, a.reps, rng), "fits": fits(ctx, a.draws, rng)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
