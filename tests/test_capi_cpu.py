"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/gdrn_b200.h declares
(no compute calls without a GPU)."""
import ctypes
import os

import pytest

from gdr_net_b200 import capi


@pytest.fixture(scope="module")
def dll():
    if not os.path.exists(capi.LIB_PATH):
        from gdr_net_b200.build import build

        build()
    return capi.C.load()


def test_header_symbols_exported(dll):
    protos = capi.parse_header()
    assert len(protos) >= 28
    for name in protos:
        assert hasattr(dll, name), name


def test_abi_version_and_error_channel(dll):
    assert dll.gdrn_abi_version() == 1
    assert isinstance(dll.gdrn_last_error(), bytes)
    assert capi.launch_count() >= 0


def test_argument_errors_do_not_need_a_gpu(dll):
    # argument validation happens on the host before any CUDA call: Cin not a multiple of 64
    rc = dll.gdrn_conv_fwd(None, None, None, None, None, None, None, None, None, None, None, 1, 8, 8, 3, 64, 64, 3, 3, 1, 1, 64, 0, 1, None)
    assert rc == -1 and b"Cin" in dll.gdrn_last_error()
    rc = dll.gdrn_gemm_fwd(None, None, None, None, None, None, None, None, None, 4, 4, 64, 100, 8, 0, 1, None)
    assert rc == -1 and b"K=" in dll.gdrn_last_error()


def test_sass_has_wgmma_and_tma():
    """The shipped library contains Hopper warpgroup tensor-core / TMA instructions (HGMMA, UTMALDG)."""
    import shutil
    import subprocess

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    for mnem in ("HGMMA", "UTMALDG"):
        assert mnem in sass, mnem
