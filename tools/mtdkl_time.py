"""mtdkl_time.py -- time one multi-task deep-kernel-learning fit step (b2gp_mtdkl_mll: MLP forward, z expanded to the GP
rows, the LCM likelihood, mll_lcm_dz_kernel, the group sum, the MLP backward) against b2gp_mll_multitask on the same
expanded z, and print one JSON line.

  step      median and minimum wall time of the whole call (it returns after its device work) over `--reps` runs after one
            warm-up, for GP rows in {2048, 8192, 16384} x both forms (multitask: one row per point; Kronecker: rows / T
            points x T tasks) x L in {1, 2}; T = 2, viMTDKL's MLP (64, 64, d = 2) at D = 64, RBF, X and y resident on the
            device as in a fit
  profile   in runs of their own, torch.profiler's device time by kernel class: mll_lcm_dz_kernel, group_sum_kernel, the
            other kernels of the step, and those of b2gp_mll_multitask; the bytes mll_lcm_dz_kernel reads (rows^2 doubles
            of K^-1 plus z, alpha and the task ids once per 32-row CTA) over its kernel time, against the data sheet's
            3.35 TB/s
Records the card's name, power limit and SM clock in the same process."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpax_b200  # noqa: E402
from gpax_b200 import _ffi  # noqa: E402
from gpax_b200.mtgp import lcm_task_matrix  # noqa: E402
from tools.dkl_time import HBM_TBPS, card, kernel_times, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rows", default="2048,8192,16384")
    ap.add_argument("--latents", default="1,2")
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    ctx = gpax_b200.default_context()
    rng = np.random.default_rng(0)
    widths, d, D, T = [64, 64, 2], 2, 64, 2
    res = {"card": card(), "widths": widths, "D": D, "T": T, "kernel": "RBF", "cases": []}
    for R in [int(v) for v in a.rows.split(",")]:
        for shared in (False, True):
            for L in [int(v) for v in a.latents.split(",")]:
                group = T if shared else 1
                N = R // group
                X = rng.uniform(-1, 1, (N, D))
                task = np.tile(np.arange(T), N) if shared else rng.integers(0, T, N)
                y = np.sin(3 * np.repeat(X[:, 0], group)) + 0.3 * task + 0.1 * rng.standard_normal(R)
                flat, i = [], D
                for w in widths:
                    flat += [rng.standard_normal(i * w) / np.sqrt(i), 0.1 * rng.standard_normal(w)]
                    i = w
                flat = np.concatenate(flat)
                theta = np.column_stack([rng.uniform(0.7, 1.2, (L, d)), np.ones(L), np.ones(L)])
                B = lcm_task_matrix(rng.normal(0, 0.7, (L, T, 1)), np.full((L, T), 0.5))
                noise = np.full(T, 0.1)
                Xd, yd = ctx.to_device(X), ctx.to_device(y)
                step = lambda: ctx.mtdkl_mll("RBF", Xd, task, yd, widths, _ffi.ACT_RELU, flat, theta, B, noise, group)  # noqa: E731
                case = {"rows": R, "form": "kronecker" if shared else "multitask", "L": L, "step": timed(step, a.reps)}
                Z = np.repeat(ctx.mlp_forward(Xd, widths, _ffi.ACT_RELU, flat)[0], group, axis=0)
                mll = lambda: ctx.mll_multitask("RBF", Z, task, y, theta, B, noise, group)   # noqa: E731
                case["mll_multitask_same_z"] = timed(mll, a.reps)
                if not a.no_profile:
                    ks, km = kernel_times(step), kernel_times(mll)
                    dz = ks.get("mll_lcm_dz_kernel", 0.0)
                    gs = ks.get("group_sum_kernel", 0.0)
                    total = sum(ks.values())
                    case["profile"] = {"mll_lcm_dz_kernel_ms": dz, "group_sum_kernel_ms": gs, "other_step_kernels_ms": total - dz - gs,
                                       "total_kernel_ms": total, "mll_multitask_kernel_ms": sum(km.values())}
                    nbytes = 8.0 * R * R + (8.0 * (d + 1) + 4.0) * R * (R // 32 + 1)
                    case["mll_lcm_dz_bytes"] = nbytes
                    case["mll_lcm_dz_tb_per_s"] = nbytes / (dz * 1e-3) / 1e12 if dz > 0 else None
                    case["mll_lcm_dz_share_of_hbm"] = case["mll_lcm_dz_tb_per_s"] / HBM_TBPS if dz > 0 else None
                res["cases"].append(case)
                Xd.free()
                yd.free()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
