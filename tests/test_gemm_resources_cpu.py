"""CPU: register budget of the GEMM kernels in the shipped library.

Every gemm_fwd_kernel / gemm_wgrad_kernel instantiation must fit in registers (no stack frame, no local-memory spills):
a spill in the forward epilogue of the 128-wide 3-pass tile is what used to keep that tile out of the library."""
import os
import re
import shutil
import subprocess

import pytest

from gdr_net_b200 import build, capi

FWD_128x3 = "_ZN4gdrn15gemm_fwd_kernelILi128ELi3EEEvNS_10GemmParamsE"


def _cuobjdump(*args):
    exe = shutil.which("cuobjdump") or os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(capi.LIB_PATH):
        build.build()
    return subprocess.run([exe, *args, capi.LIB_PATH], capture_output=True, text=True, check=True).stdout


def test_gemm_kernels_use_no_stack():
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("-res-usage")))
    gemm = {name: res for name, res in usage.items() if "gemm_fwd_kernel" in name or "gemm_wgrad_kernel" in name}
    assert FWD_128x3 in gemm
    assert sum("gemm_wgrad_kernel" in name for name in gemm) >= 2
    for name, res in gemm.items():
        assert "STACK:0 " in res and "LOCAL:0 " in res, (name, res)


def test_fwd_128x3_kernel_issues_128_wide_mma_without_local_memory():
    sass = _cuobjdump("-sass")
    bodies = re.split(r"\n\s*Function : ", sass)
    body = next(b for b in bodies if b.startswith(FWD_128x3))
    assert "HGMMA.64x128x16" in body
    assert not re.search(r"\b(LDL|STL)\b", body)


def test_outputs_beyond_32bit_offsets_are_rejected():
    # the forward epilogue addresses its output and residual planes with 32-bit element offsets
    if not os.path.exists(capi.LIB_PATH):
        build.build()
    dll = capi.C.load()
    rc = dll.gdrn_gemm_fwd(None, None, None, None, None, None, None, None, None, 1 << 20, 4, 64, 64, 4096, 0, 1, None)
    assert rc == -1 and b"32-bit" in dll.gdrn_last_error()
