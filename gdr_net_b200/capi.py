"""ctypes binding of libgdrn_b200.so.  Prototypes are parsed from include/gdrn_b200.h so the Python side
cannot drift from the C ABI.  There is NO fallback: if the library is missing or a call fails, we raise."""
from __future__ import annotations

import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "gdrn_b200.h")
LIB_PATH = os.environ.get("GDRN_LIB_PATH") or os.path.join(_HERE, "lib", "libgdrn_b200.so")  # override: A/B of two builds

_SCALARS = {"int": ctypes.c_int, "long": ctypes.c_long, "float": ctypes.c_float, "double": ctypes.c_double,
            "long long": ctypes.c_longlong}


class PoseSwitches(ctypes.Structure):
    """gdrn_pose_switches of include/gdrn_b200.h (passed by value)."""

    _fields_ = [("pm_mode", ctypes.c_int), ("pm_type", ctypes.c_int), ("pm_beta", ctypes.c_float),
                ("pm_norm_extent", ctypes.c_int), ("rot_type", ctypes.c_int), ("centroid_type", ctypes.c_int),
                ("z_type", ctypes.c_int), ("trans_type", ctypes.c_int), ("trans_disentangle", ctypes.c_int),
                ("bind_type", ctypes.c_int)]


_SCALARS["gdrn_pose_switches"] = PoseSwitches


def parse_header(path: str = HEADER) -> dict:
    """name -> (restype, [argtypes]) for every `gdrn_*` prototype in the public header."""
    txt = open(path).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    protos = {}
    for m in re.finditer(r"([A-Za-z_ ]+?\**)\s*(gdrn_\w+)\s*\(([^)]*)\)\s*;", txt):
        ret, name, args = m.group(1).strip(), m.group(2), m.group(3).strip()
        if "char" in ret:
            restype = ctypes.c_char_p
        else:
            restype = _SCALARS[ret.replace("const", "").strip()]
        argtypes = []
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                if "*" in a:
                    argtypes.append(ctypes.c_void_p)
                else:
                    typ = re.sub(r"\b\w+$", "", a.replace("const", "")).strip()
                    argtypes.append(_SCALARS[typ])
        protos[name] = (restype, argtypes)
    return protos


class GdrnError(RuntimeError):
    pass


class _Lib:
    def __init__(self):
        self._dll = None

    def load(self):
        if self._dll is not None:
            return self._dll
        if not os.path.exists(LIB_PATH):
            raise GdrnError(
                f"{LIB_PATH} not found: build it with `python -m gdr_net_b200.build` (nvcc, sm_90a). "
                "There is no CPU / PyTorch fallback for the hot path."
            )
        import torch  # noqa: F401  (loads libcudart first so the library shares torch's CUDA runtime)

        dll = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        for name, (restype, argtypes) in parse_header().items():
            fn = getattr(dll, name)  # AttributeError if the header declares something the .so lacks
            fn.restype = restype
            fn.argtypes = argtypes
        self._dll = dll
        return dll

    def __getattr__(self, name):
        dll = self.load()
        fn = getattr(dll, name)
        if fn.restype is not ctypes.c_int:
            return fn

        def checked(*args):
            rc = fn(*args)
            if rc != 0:
                raise GdrnError(f"{name} failed ({rc}): {dll.gdrn_last_error().decode()}")
            return rc

        checked.__name__ = name
        setattr(self, name, checked)
        return checked


C = _Lib()


def launch_count() -> int:
    return int(C.load().gdrn_launch_count())
