"""Where the device time of the headline posterior goes, per kernel class.

  python tools/posterior_profile.py [--opt key=value ...] [--tag NAME] [--out DIR]

Runs the bench.py workload (same make_inputs, seeds, options and call) under torch.profiler with CUDA activities, in a
run of its own with no timing taken, in two cases:
  step8   one 8-draw step on 8 streams (what bench.py times)
  draw1   one draw alone (S = 1, one stream)
and writes DIR/profile_<tag>.json: device time per (kernel, grid) and per class, and a printed table.  Kernel time is
summed over streams, so in `step8` the class sums add up to more than the step's wall time; `span_ms` is the time from
the first kernel's start to the last kernel's end.

Classes: gemm_tma (>= 1 wave: grid of one CTA per SM), gemm_tma (< 1 wave), gemm_tma_panel (the k-triangular in-place
panel solve), gemm_nt by tile configuration (panel-solve instantiations apart), trsm_strip, potrf_diag, gram, rowdot,
other.
"""
import argparse
import json
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (make_inputs and WORKLOAD of the headline workload)


def classify(name, grid, sm_count):
    if "gemm_tma_kernel" in name:
        if re.search(r"gemm_tma_kernel<\d+, \d+, true>", name):
            return "gemm_tma_panel"
        return "gemm_tma (>= 1 wave)" if grid[0] >= sm_count else "gemm_tma (< 1 wave)"
    m = re.search(r"gemm_nt_kernel<(\d+), (\d+), (\d+), (\d+), (\d+), (true|false), (\d+)(, (true|false))?>", name)
    if m:
        cfg = f"{m.group(1)}x{m.group(2)} w{m.group(3)}x{m.group(4)} s{m.group(5)}"
        return ("gemm_nt_panel " if m.group(9) == "true" else "gemm_nt ") + cfg
    for key in ("trsm_strip", "potrf_diag", "rowdot"):
        if key in name:
            return key
    if "gram" in name:
        return "gram"
    return "other"


def profile_case(ctx, ffi, S, streams, X, y, Xn, theta):
    import torch
    from torch.profiler import ProfilerActivity, profile

    w = bench.WORKLOAD
    N, d, P = w["N"], w["d"], w["P"]
    ctx.set_option("streams", streams)
    th = np.ascontiguousarray(theta[:S])
    dX, dy, dXn, dth = ctx.to_device(X), ctx.to_device(y), ctx.to_device(Xn), ctx.to_device(th)
    dmean, dvar = ctx.alloc((S, P)), ctx.alloc((S, P))
    info = np.zeros(S, dtype=np.int32)

    def step():
        ctx._check(ctx.lib.b2gp_posterior(ctx.h, ffi.KIND[w["kernel"]], dX.ptr, N, dy.ptr, 0, dXn.ptr, P, d, S, dth.ptr, 0,
                                          w["jitter"], ffi.OUT_MEAN | ffi.OUT_VAR | ffi.FLAG_DEVICE_PTRS, dmean.ptr, dvar.ptr,
                                          None, None, 0, None, info.ctypes.data, None))
        ctx.sync()

    for _ in range(3):
        step()
    assert (info == 0).all(), f"factorisation failed: info={info}"
    before = ctx.path_counts()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    after = ctx.path_counts()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    kernels = [e for e in trace["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    return kernels, {k: after[k] - before[k] for k in after}


def summarise(kernels, sm_count):
    per_kernel, per_class = {}, {}
    t0 = min(e["ts"] for e in kernels)
    t1 = max(e["ts"] + e["dur"] for e in kernels)
    total = 0.0
    for e in kernels:
        name = e["name"]
        grid = list(e.get("args", {}).get("grid", [0, 0, 0]))
        us = float(e["dur"])
        total += us
        key = f"{name} grid={grid[0]}x{grid[1]}x{grid[2]}"
        pk = per_kernel.setdefault(key, {"launches": 0, "ms": 0.0})
        pk["launches"] += 1
        pk["ms"] += us / 1e3
        cls = classify(name, grid, sm_count)
        pc = per_class.setdefault(cls, {"launches": 0, "ms": 0.0})
        pc["launches"] += 1
        pc["ms"] += us / 1e3
    for v in per_class.values():
        v["share"] = v["ms"] / (total / 1e3)
    per_kernel = dict(sorted(per_kernel.items(), key=lambda kv: -kv[1]["ms"]))
    per_class = dict(sorted(per_class.items(), key=lambda kv: -kv[1]["ms"]))
    return {"span_ms": (t1 - t0) / 1e3, "kernel_ms": total / 1e3, "launches": len(kernels), "classes": per_class,
            "kernels": per_kernel}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--opt", action="append", default=[], help="library option key=value")
    ap.add_argument("--tag", default="default")
    ap.add_argument("--out", default=".", help="output directory (default: the current directory)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("posterior_profile.py needs a CUDA device")
    from gpax_b200 import _ffi as ffi
    ctx = ffi.Context(0)
    for kv in args.opt:
        k_, v_ = kv.split("=")
        ctx.set_option(k_, int(v_))
    sm_count = ctx.device_info()["sm_count"]
    X, y, Xn, theta = bench.make_inputs(0)
    res = {"tag": args.tag, "opts": args.opt, "device": torch.cuda.get_device_name(0), "sm_count": sm_count, "cases": {}}
    for case, S, streams in (("step8", bench.WORKLOAD["S"], 8), ("draw1", 1, 1)):
        kernels, paths = profile_case(ctx, ffi, S, streams, X, y, Xn, theta)
        res["cases"][case] = summarise(kernels, sm_count)
        res["cases"][case]["paths"] = paths
    os.makedirs(args.out, exist_ok=True)
    out = os.path.join(args.out, f"profile_{args.tag}.json")
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    for case, r in res["cases"].items():
        print(f"== {args.tag} {case}: span {r['span_ms']:.2f} ms, kernel time {r['kernel_ms']:.2f} ms, {r['launches']} launches")
        for cls, v in r["classes"].items():
            print(f"   {cls:<34s} {v['launches']:6d} {v['ms']:10.3f} ms {100 * v['share']:6.2f} %")
    print("wrote", out)


if __name__ == "__main__":
    main()
