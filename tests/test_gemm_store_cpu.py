"""CPU: the shipped library holds the TMA-store forward GEMM kernel for every tile shape: gemm_fwd_tma_kernel stages its 16-bit
output tiles in shared memory and writes them with TMA stores (UTMASTG) while its MMA warpgroups go on to the next tile."""
import os
import re
import shutil
import subprocess

import pytest

from gdr_net_b200 import build, capi

INSTANTIATIONS = [(n, s) for n in (64, 128) for s in (1, 3)]


def _sass_bodies():
    exe = shutil.which("cuobjdump") or os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(capi.LIB_PATH):
        build.build()
    sass = subprocess.run([exe, "-sass", capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    return {b.split("\n", 1)[0].strip(): b for b in re.split(r"\n\s*Function : ", sass)[1:]}


def test_every_tma_kernel_instantiation_stores_with_tma():
    bodies = _sass_bodies()
    kernel = "gemm_fwd_tma_kernel"
    for n, s in INSTANTIATIONS:
        name = f"_ZN4gdrn{len(kernel)}{kernel}ILi{n}ELi{s}EEEvNS_10GemmParamsE"
        assert name in bodies, name
        assert "UTMASTG.2D" in bodies[name], name
