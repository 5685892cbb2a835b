"""The fp64 GEMM kernels issue Hopper's m16n8k4 DMMA, not the Ampere m8n8k4 shape.

On the H100 `DMMA.8x8x4` runs at half the fp64 tensor rate of the m16n8 shapes (DESIGN.md 4.3), so a kernel that falls
back to it halves the speed of the factorisation without changing a single result.  This reads the SASS of the built
library (cuobjdump -sass) and checks every instantiation of the three kernels that carry the posterior's flops."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gpax_b200", "lib", "libb200gp.so")
KERNELS = ("gemm_tma_kernel", "gemm_nt_kernel", "trsm_strip_kernel")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


def _dmma_by_function():
    out = subprocess.run([_cuobjdump(), "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = {}
            continue
        m = re.search(r"\b(DMMA\.\w+)", line)
        if cur is not None and m:
            funcs[cur][m.group(1)] = funcs[cur].get(m.group(1), 0) + 1
    return funcs


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not installed")
@pytest.mark.skipif(not os.path.exists(LIB), reason="library not built")
def test_fp64_gemm_kernels_issue_m16n8k4():
    funcs = _dmma_by_function()
    seen = {k: 0 for k in KERNELS}
    for name, dmma in funcs.items():
        kern = next((k for k in KERNELS if k in name), None)
        if kern is None:
            continue
        seen[kern] += 1
        assert dmma.get("DMMA.16x8x4", 0) > 0, (name, dmma)
        assert set(dmma) == {"DMMA.16x8x4"}, (name, dmma)
    assert all(seen.values()), seen
    # the pivot chain of the diagonal-block factorisation keeps m8n8k4 (its cost is the dependent chain, not the rate)
    assert any("potrf_diag_kernel" in n and "DMMA.8x8x4" in d for n, d in funcs.items())
