"""CPU: the 256-row forward GEMM tile (gemm_fwd_tall_kernel<128, 1>) in the shipped library: each MMA warpgroup issues two
m64n128k16 MMAs per k16 step (one per 64-row half of its 128 rows), the tile leaves through TMA stores, and its 128
accumulator registers fit without a stack frame or local memory."""
import os
import re
import shutil
import subprocess

import pytest

from gdr_net_b200 import build, capi

TALL = "_ZN4gdrn20gemm_fwd_tall_kernelILi128ELi1EEEvNS_10GemmParamsE"
K_STEPS = 64 // 16  # k16 steps per 64-deep k-block; the main loop is unrolled over them


def _cuobjdump(*args):
    exe = shutil.which("cuobjdump") or os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(capi.LIB_PATH):
        build.build()
    return subprocess.run([exe, *args, capi.LIB_PATH], capture_output=True, text=True, check=True).stdout


def test_tall_kernel_uses_no_stack():
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("-res-usage")))
    assert TALL in usage
    assert "STACK:0 " in usage[TALL] and "LOCAL:0 " in usage[TALL], usage[TALL]


def test_tall_kernel_issues_two_mmas_per_k_step_and_stores_with_tma():
    sass = _cuobjdump("-sass")
    bodies = {b.split("\n", 1)[0].strip(): b for b in re.split(r"\n\s*Function : ", sass)[1:]}
    body = bodies[TALL]
    assert len(re.findall(r"HGMMA\.64x128x16", body)) == 2 * K_STEPS
    assert "UTMASTG.2D" in body
    assert not re.search(r"\b(LDL|STL)\b", body)
