"""dkl_time.py -- time one deep-kernel-learning fit step (b2gp_dkl_mll: MLP forward, the likelihood on z, d/dz, the MLP
backward) and print one JSON line.

  step      median and minimum wall time of the whole call (it returns after its device work) over `--reps` runs after one
            warm-up, for N in {2048, 8192, 16384} x D in {64, 4096}, viDKL's MLP (64, 64, d = 2), RBF, X and y resident
            on the device as in a fit
  profile   in runs of their own, torch.profiler's device time by kernel class: the MLP GEMMs (the GEMM time of the step
            minus that of b2gp_mll on the same z), the MLP epilogues (bias + activation, its mask, column sums,
            transposes), mll_dz_kernel and the likelihood's own kernels; and the bytes mll_dz_kernel reads (N^2 doubles of
            K^-1 plus its inputs) over its kernel time, against the data sheet's 3.35 TB/s
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
from gpax_b200 import _ffi  # noqa: E402

HBM_TBPS = 3.35
EPILOGUES = ("mlp_bias_act_kernel", "mlp_act_grad_kernel", "mlp_colsum_kernel", "mlp_transpose_kernel")
GEMMS = ("gemm_nt_kernel", "gemm_tma_kernel", "oz_mma_kernel", "oz_slice_kernel")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")])) if out else {}


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": float(np.median(ts)), "min_ms": float(np.min(ts))}


def kernel_times(fn):
    """torch.profiler device time (ms, summed over launches) per kernel name during fn()"""
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
        out[base] = out.get(base, 0.0) + e.device_time_total / 1e3
    return out


def classes(step, mll):
    gem = lambda t: sum(v for k, v in t.items() if k in GEMMS)   # noqa: E731
    epi = sum(step.get(k, 0.0) for k in EPILOGUES)
    dz = step.get("mll_dz_kernel", 0.0)
    total = sum(step.values())
    return {"mlp_gemm_ms": gem(step) - gem(mll), "mlp_epilogue_ms": epi, "mll_dz_kernel_ms": dz,
            "mll_kernels_ms": total - (gem(step) - gem(mll)) - epi - dz, "total_kernel_ms": total}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="2048,8192,16384")
    ap.add_argument("--dims", default="64,4096")
    a = ap.parse_args()
    ctx = gpax_b200.default_context()
    rng = np.random.default_rng(0)
    widths, d = [64, 64, 2], 2
    theta = np.array([0.8, 1.1, 1.0, 0.1, 1.0])
    res = {"card": card(), "widths": widths, "kernel": "RBF", "cases": []}
    for N in [int(v) for v in a.sizes.split(",")]:
        for D in [int(v) for v in a.dims.split(",")]:
            X = rng.uniform(-1, 1, (N, D))
            y = np.sin(3 * X[:, 0]) + 0.1 * rng.standard_normal(N)
            flat, i = [], D
            for w in widths:
                flat += [rng.standard_normal(i * w) / np.sqrt(i), 0.1 * rng.standard_normal(w)]
                i = w
            flat = np.concatenate(flat)
            Xd, yd = ctx.to_device(X), ctx.to_device(y)
            step = lambda: ctx.dkl_mll("RBF", Xd, yd, widths, _ffi.ACT_RELU, flat, theta)   # noqa: E731
            case = {"N": N, "D": D, "step": timed(step, a.reps)}
            Z = ctx.mlp_forward(Xd, widths, _ffi.ACT_RELU, flat)[0]
            case["mll_same_z"] = timed(lambda: ctx.mll("RBF", Z, y, theta), a.reps)
            ks, km = kernel_times(step), kernel_times(lambda: ctx.mll("RBF", Z, y, theta))
            case["profile"] = classes(ks, km)
            dz_ms = ks.get("mll_dz_kernel", 0.0)
            nbytes = 8.0 * N * N + 8.0 * N * (d + 1) * (N // 32 + 1)   # K^-1 once, z and alpha per 32-row CTA
            case["mll_dz_bytes"] = nbytes
            case["mll_dz_tb_per_s"] = nbytes / (dz_ms * 1e-3) / 1e12 if dz_ms > 0 else None
            case["mll_dz_share_of_hbm"] = case["mll_dz_tb_per_s"] / HBM_TBPS if dz_ms > 0 else None
            res["cases"].append(case)
            Xd.free()
            yd.free()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
