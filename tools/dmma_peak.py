"""dmma_peak.py -- measured fp64 tensor ceiling of this GPU per DMMA instruction shape: a bare mma.sync loop on
register-resident operands, one CTA of eight warps per SM, no shared memory, no epilogue (dmma_peak_kernel).

  python tools/dmma_peak.py [OUT.json]

Prints one JSON object: the card, its power limit and SM clocks (nvidia-smi, read-only) and, per shape, TFLOP/s and
FMA/clk/SM at the SM clock read right after the timed launches."""
import ctypes as C
import json
import subprocess
import sys

sys.path.insert(0, ".")
from gpax_b200 import _ffi  # noqa: E402

SHAPES = ["m8n8k4", "m16n8k4", "m16n8k8", "m16n8k16"]


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [f.strip() for f in out.split(",")]
    except Exception as e:  # noqa: BLE001
        return [f"nvidia-smi unavailable: {e}"]


def main():
    ctx = _ffi.Context(0)
    fn = ctx.lib.b2gp_debug_dmma_peak
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    name, power_limit, max_mhz = (smi("name,power.limit,clocks.max.sm") + [None, None])[:3]
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = {"card": name, "power_limit_w": power_limit, "sm_max_mhz": max_mhz, "sm_count": sms, "shapes": {}}
    for shape, label in enumerate(SHAPES):
        tf, ms = C.c_double(), C.c_double()
        # the same flops for every shape, ~70 ms per launch at 128 FMA/clk/SM and 1.98 GHz: long enough that launch
        # overhead does not show
        iters = (1 << 20) * 256 // (8 * 8 * 4 if shape == 0 else 16 * 8 * (4 << (shape - 1)))
        rc = fn(ctx.h, shape, iters, 5, C.byref(tf), C.byref(ms))
        assert rc == 0, ctx.lib.b2gp_last_error(ctx.h)
        mhz = smi("clocks.sm")[0]
        try:
            fma_clk_sm = tf.value * 1e12 / 2 / sms / (float(mhz) * 1e6)
        except ValueError:
            fma_clk_sm = None
        res["shapes"][label] = {"tflops": tf.value, "ms": ms.value, "iters": iters, "sm_mhz_after": mhz, "fma_per_clk_per_sm": fma_clk_sm}
    print(json.dumps(res))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
